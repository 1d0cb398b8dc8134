"""Learner-side helpers of the reference's ``utils.py`` that ``train_impala.py`` touches.

  check_properties   utils.py:34-45  (config validation before the learner is built)
  copy_src_to_dst    utils.py:6-22   (learner -> actor variable copy; here a callable shim)

  UnrolledTrajectory utils.py:80-119  (the actor-side accumulator whose ``extract()`` feeds ``FIFOQueue.append_to_queue``,
                                       train_impala.py:117,165-189: closes the actor -> ring -> learner loop)
  impala_env_step    (new) the IMPALA actor's rule for one environment step, shared by actor.VectorActor and the
                     worker processes of actor_server.EnvWorkerPool; it is the A3C actor's rule too, and the workers of
                     actor_server.A3CEnvWorkerPool step under it
  r2d2_env_step      (new) the R2D2 actor's rule for one environment step, shared by actor.R2D2VectorActor and the
                     worker processes of actor_server.R2D2EnvWorkerPool
"""
import collections

START_LIVES = 5   # the reference actor's life counter starts (and restarts after every episode) at 5


def impala_env_step(env, action, available_action, stats, i, max_prob, task=None):
    """One step of environment i under the IMPALA actor's rules (train_impala.py:150-175).  ``stats`` holds the
    per-environment lists ``lives``, ``episode``, ``score``, ``episode_step`` and ``total_max_prob``; ``max_prob`` is
    the largest probability of the policy the action was drawn from.

      - the environment steps with ``action % available_action`` (the trajectory stores the action unmodified);
      - a lost life (``info['ale.lives']`` changed) is stored as reward -1 and done=True; the score keeps the raw reward;
      - at an episode's end the environment is reset and the caller sets previous action, h and c back to 0.

    Returns (next_state, reward, done, state, finished): env.step's frame, the reward and done flag the trajectory
    stores, the frame the next action is for (a fresh episode's first frame after an episode end), and the finished
    episode's dict of task (``task``, default i), episode, score, episode_step and prob (mean max probability) -- the
    values train_impala.py:170-172 logs -- or None."""
    stats.episode_step[i] += 1
    stats.total_max_prob[i] += float(max_prob)
    next_state, reward, done, info = env.step(action % available_action)
    stats.score[i] += reward
    if stats.lives[i] != info["ale.lives"]:
        r, d = -1.0, True
    else:
        r, d = reward, False
    stats.lives[i] = info["ale.lives"]
    state, finished = next_state, None
    if done:
        finished = dict(task=i if task is None else task, episode=stats.episode[i], score=stats.score[i],
                        episode_step=stats.episode_step[i], prob=stats.total_max_prob[i] / stats.episode_step[i])
        stats.episode[i] += 1
        stats.score[i], stats.episode_step[i], stats.total_max_prob[i] = 0.0, 0, 0.0
        state = env.reset()
        stats.lives[i] = START_LIVES
    return next_state, r, d, state, finished


def r2d2_env_step(env, action, stats, i, q_action, task=None):
    """One step of environment i under the R2D2 actor's rules (train_r2d2.py:196-235).  ``stats`` holds the
    per-environment lists ``lives``, ``episode``, ``epsilon``, ``score``, ``episode_step`` and ``episode_q_value``;
    ``q_action`` is q[action] of the act that chose the action.

      - the environment steps with the raw action (the R2D2 actor applies no ``% available_action``);
      - ``lives`` is only set back to 5 at an episode's end, never after a life loss, so every step after the first
        life loss of an episode is stored as reward -1 and done=True (the reference's behaviour); the score keeps the
        raw reward;
      - at an episode's end epsilon becomes 1 / (0.01 episode + 1), the environment is reset, and the caller sets the
        previous action, h and c back to 0.  episode_step and the summed q of the logged average are never reset.

    Returns (next_state, reward, done, state, finished): env.step's frame, the reward and done flag the sequence
    stores, the frame the next action is for (a fresh episode's first frame after an episode end), and the finished
    episode's dict of task (``task``, default i), episode, score, epsilon, episode_step and avg_q_value -- the values
    train_r2d2.py:227-230 logs -- or None."""
    stats.episode_q_value[i] += float(q_action)
    stats.episode_step[i] += 1
    next_state, reward, done, info = env.step(action)
    stats.score[i] += reward
    if stats.lives[i] != info["ale.lives"]:
        r, d = -1, True
    else:
        r, d = reward, False
    state, finished = next_state, None
    if done:
        finished = dict(task=i if task is None else task, episode=stats.episode[i], score=stats.score[i],
                        epsilon=stats.epsilon[i], episode_step=stats.episode_step[i],
                        avg_q_value=stats.episode_q_value[i] / stats.episode_step[i])
        stats.episode[i] += 1
        stats.score[i] = 0
        stats.epsilon[i] = 1.0 / (0.01 * stats.episode[i] + 1)
        state = env.reset()
        stats.lives[i] = START_LIVES
    return next_state, r, d, state, finished


def check_properties(data):
    """Same five checks as the reference, raising AssertionError on a bad config."""
    n_actors = data['num_actors']
    avail, envs = data['available_action'], data['env']
    assert all(data['model_output'] >= a for a in avail), "available_action exceeds model_output"
    assert n_actors == len(avail), "num_actors != len(available_action)"
    assert n_actors == len(envs), "num_actors != len(env)"
    assert len(avail) == len(envs), "len(available_action) != len(env)"
    assert data['reward_clipping'] in ['abs_one', 'soft_asymmetric'], "unknown reward_clipping"


def copy_src_to_dst(from_scope, to_scope):
    """Returns a zero-argument callable that copies the variables of agent `from_scope` into agent
    `to_scope` (what running the reference's assign ops does)."""
    from .agent import impala

    def run():
        dst = impala._AGENTS.get(to_scope)
        if dst is not None:
            dst.parameter_sync()
    return run


class _Accumulator:
    """Per-actor accumulator of one unroll: ``initialize()`` empties it, ``append(...)`` adds one step."""
    _FIELDS = ()

    def __init__(self):
        self.trajectory_data = collections.namedtuple('trajectory_data', list(self._FIELDS))

    def initialize(self):
        self.unroll_data = self.trajectory_data(*[[] for _ in self._FIELDS])

    def _add(self, values):
        for field, value in zip(self.unroll_data, values):
            field.append(value)


class UnrolledA3CTrajectory(_Accumulator):
    """utils.py:47-78: the A3C actor's unroll; ``extract()`` stacks every field (train_a3c.py feeds it to A3CFIFOQueue)."""
    _FIELDS = ('state', 'next_state', 'reward', 'done', 'action', 'previous_action')

    def append(self, state, next_state, previous_action, action, reward, done):
        self._add((state, next_state, reward, done, action, previous_action))

    def extract(self):
        import numpy as np
        return {k: np.stack(v) for k, v in self.unroll_data._asdict().items()}


class UnrolledTrajectory:
    """utils.py:80-119: per-actor accumulator of one unroll; ``extract()`` returns the nine per-step lists that
    ``FIFOQueue.append_to_queue`` takes (train_impala.py:178-189)."""

    def __init__(self):
        self.trajectory_data = collections.namedtuple(
            'trajectory_data',
            ['state', 'next_state', 'reward', 'done', 'action', 'behavior_policy', 'previous_action',
             'initial_h', 'initial_c'])

    def initialize(self):
        self.unroll_data = self.trajectory_data(*[[] for _ in range(9)])

    def append(self, state, next_state, reward, done, action, behavior_policy, previous_action, initial_h, initial_c):
        for field, value in zip(self.unroll_data, (state, next_state, reward, done, action, behavior_policy,
                                                   previous_action, initial_h, initial_c)):
            field.append(value)

    def extract(self):
        return dict(self.unroll_data._asdict())
