"""Vector actors: the actor branches of ``train_impala.py:117-194`` (VectorActor, on one NativePolicy), of
``train_r2d2.py:167-251`` (R2D2VectorActor, on one NativeR2D2Policy), of ``train_apex.py:157-231`` (ApexVectorActor, on
one NativeApexPolicy) and of ``train_a3c.py:112-183`` (A3CVectorActor, on one NativeA3CPolicy) for N environments in
lockstep.

VectorActor: each environment is its own actor task ``i`` (what ``FLAGS.task`` selects in the reference).  Per unroll:

  - one parameter sync through ``learner.sync_policy(policy)`` (the learner-side ``impala.Agent``; device to device
    when it has a CUDA learner);
  - ``trajectory`` batched ``policy.act`` calls: one forward over all N environments, the actions drawn on the GPU
    from the same global ``np.random`` stream the reference's ``np.random.choice`` reads;
  - every environment steps under ``utils.impala_env_step`` (the rule the worker processes of
    ``actor_server.EnvWorkerPool`` follow too): ``action % available_action[i]``, the trajectory stores the action
    unmodified (SURVEY.md App. D); a lost life (``info['ale.lives']`` changed) is stored as reward -1 and done=True,
    the score keeps the raw reward; at an episode's end the environment is reset, and previous action, h and c go
    back to 0;
  - every environment's ``utils.UnrolledTrajectory`` goes to ``queue.append_to_queue(task=i, ...)``; with a
    ``DeviceFIFOQueue`` the acts go through a recorder of the policy instead (``NativePolicy.recorder``), which keeps
    the trajectories on the GPU, and the unroll ends with one ``commit`` of the rewards and done flags of all N
    environments, in environment order.
"""
import numpy as np

from . import utils
from .distributed_queue import buffer_queue
from .utils import START_LIVES


class VectorActor:
    def __init__(self, policy, envs, queue, trajectory, available_action, learner=None):
        self.policy, self.envs, self.queue, self.learner = policy, list(envs), queue, learner
        self.trajectory = int(trajectory)
        self.available_action = [int(a) for a in available_action]
        n = len(self.envs)
        if not 1 <= n <= policy.max_batch:
            raise ValueError("%d environments, the policy serves 1..%d per call" % (n, policy.max_batch))
        if len(self.available_action) != n:
            raise ValueError("available_action has %d entries for %d environments" % (len(self.available_action), n))
        L = policy.L
        self.states = [env.reset() for env in self.envs]
        self.previous_action = np.zeros(n, np.int32)
        self.h = np.zeros((n, L), np.float32)
        self.c = np.zeros((n, L), np.float32)
        self.lives = [START_LIVES] * n
        self.episode = [0] * n
        self.score = [0.0] * n
        self.episode_step = [0] * n
        self.total_max_prob = [0.0] * n
        self.recorder = None
        if isinstance(queue, buffer_queue.DeviceFIFOQueue):
            self._check_device_queue(queue)
            self.recorder = policy.recorder(queue, n)

    def _check_device_queue(self, queue):
        p = self.policy
        if queue.trajectory != self.trajectory:
            raise ValueError("queue records trajectories of %d steps, the actor unrolls %d"
                             % (queue.trajectory, self.trajectory))
        if queue.output_size != p.A:
            raise ValueError("queue has num_action %d, the policy %d" % (queue.output_size, p.A))
        if queue.lstm_size != p.L or tuple(queue.input_shape) != tuple(p.input_shape):
            raise ValueError("queue stores %s frames and lstm %d, the policy takes %s and %d"
                             % (tuple(queue.input_shape), queue.lstm_size, tuple(p.input_shape), p.L))
        if queue.device != p.device:
            raise ValueError("queue is on device %d, the policy on device %d" % (queue.device, p.device))
        n = len(self.envs)
        if n > queue.max_rows:
            raise ValueError("%d environments per commit, the queue takes at most %d at once" % (n, queue.max_rows))

    def run_unroll(self):
        """One unroll of `trajectory` steps for every environment, pushed to the queue.  Returns the episodes that
        finished during it: dicts of task, episode, score, episode_step and prob (mean max probability), the values
        train_impala.py:170-172 logs."""
        if self.learner is not None:
            self.learner.sync_policy(self.policy)
        n = len(self.envs)
        rec = self.recorder
        if rec is None:
            trajs = [utils.UnrolledTrajectory() for _ in range(n)]
            for t in trajs:
                t.initialize()
            act = self.policy.act
        else:
            rec.reset()   # an unroll that raised half-way left its steps behind: start this one at step 0
            rewards = np.zeros((n, self.trajectory), np.float32)
            dones = np.zeros((n, self.trajectory), np.bool_)
            act = rec.act
        finished = []
        for step in range(self.trajectory):
            out = act(np.stack(self.states), self.previous_action, self.h, self.c)
            action, policy, max_prob = out["action"], out["policy"], out["max_prob"]
            # fresh copies: rows already stored in a trajectory, and the arrays act returned, are never written again
            next_pa, next_h, next_c = action.astype(np.int32), out["h"].copy(), out["c"].copy()
            for i, env in enumerate(self.envs):
                a = int(action[i])
                next_state, r, d, state, episode = utils.impala_env_step(env, a, self.available_action[i], self, i,
                                                                         max_prob[i])
                if rec is None:
                    trajs[i].append(state=self.states[i], next_state=next_state, reward=r, done=d, action=a,
                                    behavior_policy=policy[i], previous_action=int(self.previous_action[i]),
                                    initial_h=self.h[i], initial_c=self.c[i])
                else:   # the rest of the step is on the device already
                    rewards[i, step], dones[i, step] = r, d
                self.states[i] = state
                if episode is not None:
                    finished.append(episode)
                    next_pa[i] = 0
                    next_h[i] = 0.0
                    next_c[i] = 0.0
            self.previous_action, self.h, self.c = next_pa, next_h, next_c
        if rec is not None:
            rec.commit(rewards, dones)
            return finished
        for i, t in enumerate(trajs):
            u = t.extract()
            self.queue.append_to_queue(
                task=i, unrolled_state=u["state"], unrolled_next_state=u["next_state"], unrolled_reward=u["reward"],
                unrolled_done=u["done"], unrolled_behavior_policy=u["behavior_policy"], unrolled_action=u["action"],
                unrolled_previous_action=u["previous_action"], unrolled_previous_h=u["initial_h"],
                unrolled_previous_c=u["initial_c"])
        return finished


class R2D2VectorActor:
    """The actor branch of ``train_r2d2.py:167-251`` for N environments in lockstep on one NativeR2D2Policy; each
    environment is its own actor task ``i``.  Per unroll:

      - every environment's ``R2D2TrajectoryBuffer.init()``, then one ``learner.sync_policy(policy)`` (the
        learner-side ``r2d2.Agent``; device to device when it has a CUDA learner);
      - ``seq_len`` batched ``policy.act`` calls with each environment's epsilon: the explore draws of environments
        0..n-1 from the global ``np.random`` stream, in that order, then every environment steps under
        ``utils.r2d2_env_step`` (the rule the worker processes of ``actor_server.R2D2EnvWorkerPool`` follow too), in
        order 0..n-1, with the raw action (the R2D2 actor applies no ``% available_action``);
      - ``lives`` is only ever set back to 5 by an episode reset, never after a life loss, so every step after the
        first life loss of an episode is stored as reward -1 and done=True (the reference's behaviour, SURVEY.md
        App. D); the score keeps the raw reward;
      - at an episode's end epsilon becomes 1 / (0.01 episode + 1), and the environment, the previous action, h, c
        and lives are reset.  episode_step and the summed q of the logged average are never reset, as in the
        reference;
      - every environment's trajectory goes to ``queue.append_to_queue(task=i, ...)``; with an
        ``R2D2DeviceFIFOQueue`` the acts go through a recorder of the policy instead (``NativeR2D2Policy.recorder``),
        which keeps the sequences on the GPU, and the unroll ends with one ``commit`` of the rewards and done flags of
        all N environments, in environment order.
    At n = 1 this is the reference actor's loop, including the order of its ``np.random`` draws.
    """

    def __init__(self, policy, envs, queue, seq_len, learner=None):
        self.policy, self.envs, self.queue, self.learner = policy, list(envs), queue, learner
        self.seq_len = int(seq_len)
        n = len(self.envs)
        if not 1 <= n <= policy.max_batch:
            raise ValueError("%d environments, the policy serves 1..%d per call" % (n, policy.max_batch))
        L = policy.L
        if learner is not None and getattr(learner, "lstm_size", L) != L:
            raise ValueError("the learner has lstm_size %d, the policy %d: the policy engine syncs from a learner of its "
                             "own width" % (learner.lstm_size, L))
        self.buffers = [buffer_queue.R2D2TrajectoryBuffer(seq_len=self.seq_len) for _ in range(n)]
        self.states = [env.reset() for env in self.envs]
        self.previous_action = np.zeros(n, np.int32)
        self.h = np.zeros((n, L), np.float32)
        self.c = np.zeros((n, L), np.float32)
        self.lives = [START_LIVES] * n
        self.episode = [0] * n
        self.epsilon = [1.0] * n
        self.score = [0.0] * n
        self.episode_step = [0] * n
        self.episode_q_value = [0.0] * n
        self.recorder = None
        if isinstance(queue, buffer_queue.R2D2DeviceFIFOQueue):
            self._check_device_queue(queue)
            self.recorder = policy.recorder(queue, n)

    def _check_device_queue(self, queue):
        p = self.policy
        if queue.seq_len != self.seq_len:
            raise ValueError("queue records sequences of %d steps, the actor unrolls %d" % (queue.seq_len, self.seq_len))
        if queue.output_size != p.A:
            raise ValueError("queue has num_action %d, the policy %d" % (queue.output_size, p.A))
        if queue.lstm_size != p.L or tuple(queue.input_shape) != tuple(p.input_shape):
            raise ValueError("queue stores %s frames and lstm %d, the policy takes %s and %d"
                             % (tuple(queue.input_shape), queue.lstm_size, tuple(p.input_shape), p.L))
        if queue.device != p.device:
            raise ValueError("queue is on device %d, the policy on device %d" % (queue.device, p.device))
        n = len(self.envs)
        if n > queue.max_rows:
            raise ValueError("%d environments per commit, the queue takes at most %d at once" % (n, queue.max_rows))

    def run_unroll(self):
        """One unroll of `seq_len` steps for every environment, pushed to the queue.  Returns the episodes that
        finished during it: dicts of task, episode, score, epsilon, episode_step and avg_q_value, the values
        train_r2d2.py:227-230 logs."""
        n = len(self.envs)
        rec = self.recorder
        if rec is None:
            for b in self.buffers:
                b.init()
            act = self.policy.act
        else:
            rec.reset()   # an unroll that raised half-way left its steps behind: start this one at step 0
            rewards = np.zeros((n, self.seq_len), np.float32)
            dones = np.zeros((n, self.seq_len), np.bool_)
            act = rec.act
        if self.learner is not None:
            self.learner.sync_policy(self.policy)
        finished = []
        for step in range(self.seq_len):
            out = act(np.stack(self.states), self.previous_action, self.h, self.c, epsilon=np.array(self.epsilon))
            action, q_action = out["action"], out["q_action"]
            # fresh copies: rows already stored in a trajectory, and the arrays act returned, are never written again
            next_pa, next_h, next_c = action.astype(np.int32), out["h"].copy(), out["c"].copy()
            for i, env in enumerate(self.envs):
                a = int(action[i])
                _, r, d, state, episode = utils.r2d2_env_step(env, a, self, i, q_action[i])
                if rec is None:
                    self.buffers[i].append(state=self.states[i], previous_action=int(self.previous_action[i]),
                                           action=a, reward=r, done=d, initial_h=self.h[i], initial_c=self.c[i])
                else:   # the rest of the step is on the device already
                    rewards[i, step], dones[i, step] = r, d
                self.states[i] = state
                if episode is not None:
                    finished.append(episode)
                    next_pa[i] = 0
                    next_h[i] = 0.0
                    next_c[i] = 0.0
            self.previous_action, self.h, self.c = next_pa, next_h, next_c
        if rec is not None:
            rec.commit(rewards, dones)
            return finished
        for i, b in enumerate(self.buffers):
            u = b.extract()
            self.queue.append_to_queue(
                task=i, unrolled_state=u["state"], unrolled_previous_action=u["previous_action"],
                unrolled_action=u["action"], unrolled_reward=u["reward"], unrolled_done=u["done"],
                unrolled_previous_h=u["initial_h"], unrolled_previous_c=u["initial_c"])
        return finished


class ApexVectorActor:
    """The actor branch of ``train_apex.py:157-231`` for N environments in lockstep on one NativeApexPolicy; each
    environment is its own actor task ``i``.  Per unroll (``trajectory`` steps):

      - one ``learner.sync_policy(policy)`` (the learner-side ``apex.Agent``; device to device when it has a CUDA
        learner);
      - ``trajectory`` batched ``policy.act`` calls with each environment's epsilon: the explore draws of environments
        0..n-1 from the global ``np.random`` stream, in that order; then, environment by environment, ``env.step`` with
        ``action % available_action[i]`` (the buffer stores the raw action), the append to its ``LocalBuffer(1e4)``
        and, once the buffer holds more than 3 ``trajectory`` transitions, a ``sample(trajectory)`` (a
        ``np.random.permutation`` draw) pushed to ``queue.append_to_queue(task=i, ...)`` -- every step from then on.
        With an ``ApexDeviceFIFOQueue`` the buffers are one ``DeviceLocalBuffers`` on the GPU instead: the
        environment loop makes the same draws at the same points, and after it one ``append`` of all n rows and one
        ``push`` per draw, in environment order, fill the queue on the device with the same records (only the moment
        a full queue blocks moves to after the environment loop);
      - every environment steps under ``utils.apex_env_step`` (the rule the worker processes of
        ``actor_server.ApexEnvWorkerPool`` follow too): a lost life (``info['ale.lives']`` changed) is stored as reward
        -1 and done=True; the score keeps the raw reward; ``lives`` follows ``info['ale.lives']`` after every step;
      - at an episode's end epsilon becomes 1 / (0.05 episode + 1), and the environment, the previous action and
        lives (5) are reset.  ``episode_step`` is reset, the summed ``q[action]`` behind the logged ratio is not (the
        reference's behaviour, SURVEY.md App. D).
    At n = 1 this is the reference actor's loop, including the order of its ``np.random`` draws.
    """

    def __init__(self, policy, envs, queue, trajectory, available_action, learner=None, buffer_capacity=int(1e4)):
        self.policy, self.envs, self.queue, self.learner = policy, list(envs), queue, learner
        self.trajectory = int(trajectory)
        self.available_action = [int(a) for a in available_action]
        n = len(self.envs)
        if not 1 <= n <= policy.max_batch:
            raise ValueError("%d environments, the policy serves 1..%d per call" % (n, policy.max_batch))
        if len(self.available_action) != n:
            raise ValueError("available_action has %d entries for %d environments" % (len(self.available_action), n))
        self.device_buffers = None
        if isinstance(queue, buffer_queue.ApexDeviceFIFOQueue):
            self._check_device_queue(queue)
            self.buffers = None
            self.device_buffers = buffer_queue.DeviceLocalBuffers(n, buffer_capacity, policy.A, policy.device)
        else:
            self.buffers = [buffer_queue.LocalBuffer(capacity=buffer_capacity) for _ in range(n)]
        self.states = [env.reset() for env in self.envs]
        self.previous_action = np.zeros(n, np.int32)
        self.lives = [START_LIVES] * n
        self.episode = [0] * n
        self.epsilon = [1.0] * n
        self.score = [0.0] * n
        self.episode_step = [0] * n
        self.total_max_prob = [0.0] * n

    def _check_device_queue(self, queue):
        p = self.policy
        if queue.trajectory != self.trajectory:
            raise ValueError("queue records samples of %d transitions, the actor samples %d"
                             % (queue.trajectory, self.trajectory))
        if queue.output_size != p.A:
            raise ValueError("queue has num_action %d, the policy %d" % (queue.output_size, p.A))
        if queue.device != p.device:
            raise ValueError("queue is on device %d, the policy on device %d" % (queue.device, p.device))

    def run_unroll(self):
        """One unroll of `trajectory` steps for every environment.  Returns the episodes that finished during it:
        dicts of task, episode, score, epsilon, episode_step and total_max_prob (the logged ratio: the running sum of
        q[action] over episode_step), the values train_apex.py:215-220 logs."""
        if self.learner is not None:
            self.learner.sync_policy(self.policy)
        finished = []
        T = self.trajectory
        db = self.device_buffers
        n = len(self.envs)
        for _ in range(T):
            out = self.policy.act(np.stack(self.states), self.previous_action, epsilon=np.array(self.epsilon))
            action, q_action = out["action"], out["q_action"]
            next_pa = action.astype(np.int32)
            if db is not None:
                # every buffer's length after this step's append, and the rows of that append
                length = min(len(db) + 1, db.capacity)
                rows = dict(state=list(self.states), next_state=[None] * n, reward=np.zeros(n, np.float32),
                            done=np.zeros(n, np.bool_))
                draws = []
            for i, env in enumerate(self.envs):
                a = int(action[i])
                next_state, r, d, state, episode = utils.apex_env_step(env, a, self.available_action[i], self, i,
                                                                       q_action[i])
                if db is None:
                    buf = self.buffers[i]
                    buf.append(state=self.states[i], done=d, reward=r, next_state=next_state,
                               previous_action=int(self.previous_action[i]), action=a)
                else:
                    rows["next_state"][i], rows["reward"][i], rows["done"][i] = next_state, r, d
                self.states[i] = state
                if db is not None:
                    if length > 3 * T:   # LocalBuffer.sample's draw, at the same point of the stream
                        draws.append((i, np.random.permutation(length)[:T]))
                elif len(buf) > 3 * T:
                    u = buf.sample(T)
                    self.queue.append_to_queue(
                        task=i, unrolled_state=u["state"], unrolled_next_state=u["next_state"],
                        unrolled_previous_action=u["previous_action"], unrolled_action=u["action"],
                        unrolled_reward=u["reward"], unrolled_done=u["done"])
                if episode is not None:
                    finished.append(episode)
                    next_pa[i] = 0
            if db is not None:
                db.append(np.stack(rows["state"]), np.stack(rows["next_state"]), self.previous_action, action,
                          rows["reward"], rows["done"])
                for i, order in draws:   # a full queue blocks here, after the environment loop
                    db.push(self.queue, i, order)
            self.previous_action = next_pa
        return finished


class A3CVectorActor:
    """The actor branch of ``train_a3c.py:112-183`` for N environments in lockstep on one NativeA3CPolicy; each
    environment is its own actor task ``i``.  Per unroll (``trajectory`` steps):

      - every environment's ``UnrolledA3CTrajectory.initialize()``, then one ``learner.sync_policy(policy)`` (the
        learner-side ``a3c.Agent``; device to device when it has a CUDA learner);
      - ``trajectory`` batched ``policy.act`` calls: ``np.random.random_sample(n)`` from the global stream (row i's
        draw is the one the reference's ``np.random.choice(A, p=policy)`` reads), the actions picked on the GPU; then,
        environment by environment, ``env.step`` with ``action % available_action[i]`` (the trajectory stores the raw
        action);
      - a lost life (``info['ale.lives']`` changed) is stored as reward -1 and done=True; the score keeps the raw
        reward; ``lives`` follows ``info['ale.lives']`` after every step;
      - at an episode's end the environment, the previous action and lives (5) are reset, and so are the score,
        ``episode_step`` and the summed ``policy[action]`` behind the logged "prob";
      - every environment's trajectory goes to ``queue.append_to_queue(task=i, ...)``; with an
        ``A3CDeviceFIFOQueue`` the acts go through a recorder of the policy instead (``NativeA3CPolicy.recorder``),
        which keeps the unrolls on the GPU, and the unroll ends with one ``commit`` of the rewards, done flags and
        final next_state frames of all N environments, in environment order.  No host trajectory is kept.
    At n = 1 this is the reference actor's loop, including the order of its ``np.random`` draws.
    """

    def __init__(self, policy, envs, queue, trajectory, available_action, learner=None):
        self.policy, self.envs, self.queue, self.learner = policy, list(envs), queue, learner
        self.trajectory = int(trajectory)
        self.available_action = [int(a) for a in available_action]
        n = len(self.envs)
        if not 1 <= n <= policy.max_batch:
            raise ValueError("%d environments, the policy serves 1..%d per call" % (n, policy.max_batch))
        if len(self.available_action) != n:
            raise ValueError("available_action has %d entries for %d environments" % (len(self.available_action), n))
        self.trajs = [utils.UnrolledA3CTrajectory() for _ in range(n)]
        self.states = [env.reset() for env in self.envs]
        self.previous_action = np.zeros(n, np.int32)
        self.lives = [START_LIVES] * n
        self.episode = [0] * n
        self.score = [0.0] * n
        self.episode_step = [0] * n
        self.total_max_prob = [0.0] * n
        self.recorder = None
        if isinstance(queue, buffer_queue.A3CDeviceFIFOQueue):
            self._check_device_queue(queue)
            self.trajs = None
            self.recorder = policy.recorder(queue, n)

    def _check_device_queue(self, queue):
        p = self.policy
        if queue.trajectory != self.trajectory:
            raise ValueError("queue records unrolls of %d steps, the actor unrolls %d" % (queue.trajectory,
                                                                                        self.trajectory))
        if queue.output_size != p.A:
            raise ValueError("queue has num_action %d, the policy %d" % (queue.output_size, p.A))
        if queue.device != p.device:
            raise ValueError("queue is on device %d, the policy on device %d" % (queue.device, p.device))
        n = len(self.envs)
        if n > queue.max_rows:
            raise ValueError("%d environments per commit, the queue takes at most %d at once" % (n, queue.max_rows))

    def run_unroll(self):
        """One unroll of `trajectory` steps for every environment, pushed to the queue.  Returns the episodes that
        finished during it: dicts of task, episode, prob (the mean policy[action]), score and episode_step, the values
        train_a3c.py:162-165 logs."""
        n = len(self.envs)
        rec = self.recorder
        if rec is None:
            for t in self.trajs:
                t.initialize()
        else:
            rec.reset()   # an unroll that raised half-way left its steps behind: start this one at step 0
            rewards = np.zeros((n, self.trajectory), np.float32)
            dones = np.zeros((n, self.trajectory), np.bool_)
            next_states = None   # env.step's frames of the previous step
        if self.learner is not None:
            self.learner.sync_policy(self.policy)
        finished = []
        for step in range(self.trajectory):
            if rec is None:
                out = self.policy.act(np.stack(self.states), self.previous_action)
            else:
                out = rec.act(np.stack(self.states), self.previous_action, previous_next_state=next_states)
                next_states = [None] * n
            action, max_prob = out["action"], out["max_prob"]
            next_pa = action.astype(np.int32)
            for i, env in enumerate(self.envs):
                a = int(action[i])
                self.episode_step[i] += 1
                self.total_max_prob[i] += float(max_prob[i])
                next_state, reward, done, info = env.step(a % self.available_action[i])
                self.score[i] += reward
                if self.lives[i] != info["ale.lives"]:
                    r, d = -1, True
                else:
                    r, d = reward, False
                if rec is None:
                    self.trajs[i].append(state=self.states[i], next_state=next_state,
                                         previous_action=int(self.previous_action[i]), action=a, reward=r, done=d)
                else:   # state, the actions and (from the next act on) next_state are on the device already
                    rewards[i, step], dones[i, step] = r, d
                    next_states[i] = next_state
                self.states[i] = next_state
                self.lives[i] = info["ale.lives"]
                if done:
                    finished.append(dict(task=i, episode=self.episode[i],
                                         prob=self.total_max_prob[i] / self.episode_step[i], score=self.score[i],
                                         episode_step=self.episode_step[i]))
                    self.episode[i] += 1
                    self.score[i] = 0
                    self.episode_step[i] = 0
                    self.total_max_prob[i] = 0
                    self.states[i] = env.reset()
                    next_pa[i] = 0
                    self.lives[i] = START_LIVES
            self.previous_action = next_pa
        if rec is not None:
            rec.commit(rewards, dones, np.stack(next_states))
            return finished
        for i, t in enumerate(self.trajs):
            u = t.extract()
            self.queue.append_to_queue(
                task=i, unrolled_state=u["state"], unrolled_next_state=u["next_state"],
                unrolled_previous_action=u["previous_action"], unrolled_action=u["action"],
                unrolled_reward=u["reward"], unrolled_done=u["done"])
        return finished
