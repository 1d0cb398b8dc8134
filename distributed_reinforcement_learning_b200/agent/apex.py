"""H100-native stand-in for the reference's ``agent/apex.py``: same constructor kwargs, same methods, same return
values -- so the learner branch of ``train_apex.py:82-155`` runs on it unchanged -- with the TF1 graph +
``tf.Session`` replaced by the CUDA Ape-X learner behind the C-ABI (``drl_apex_*``).

  Agent.__init__              agent/apex.py:12-76
  Agent.target_to_main        agent/apex.py:78-79   (assigns target <- main, as utils.main_to_target does)
  Agent.parameter_sync        agent/apex.py:81-82   (learner -> this agent's variables)
  Agent.set_session           agent/apex.py:84-86   (also initialises every variable, like the reference)
  Agent.get_policy_and_action agent/apex.py:88-102
  Agent.get_td_error          agent/apex.py:116-133
  Agent.distributed_train     agent/apex.py:135-154 -> (loss, td_error)
  Agent.train                 agent/apex.py:156-168
  Agent.sync_policy           parameter_sync into a NativeApexPolicy (actor.py: ApexVectorActor)
  Agent.device_memory         a DeviceMemory: the replay memory of train_apex.py:87 on the GPU (apex_replay.py);
                              DeviceMemory.add_from_queue ingests a record of an ApexDeviceFIFOQueue without a host copy
  Agent.train_from_memory     Memory.sample + np.stack + distributed_train + Memory.update (train_apex.py:118-154)
                              as one device-resident step -> (loss, td_error)
"""
import os
import random
import threading

import numpy as np

from .. import dp
from ..apex_learner import MAIN, TARGET, NativeApexLearner
from ..apex_replay import NativeApexReplay
from ..model import apex_value

_AGENTS = {}


class Agent:

    def __init__(self, input_shape, num_action,
                 discount_factor, gradient_clip_norm, reward_clipping,
                 start_learning_rate, end_learning_rate, learning_frame,
                 model_name, learner_name):
        self.input_shape = list(input_shape)
        self.num_action = num_action
        self.discount_factor = discount_factor
        self.gradient_clip_norm = gradient_clip_norm
        self.reward_clipping = reward_clipping
        self.start_learning_rate = start_learning_rate
        self.end_learning_rate = end_learning_rate
        self.learning_frame = learning_frame
        self.model_name = model_name
        self.learner_name = learner_name
        self.device = int(os.environ.get("LOCAL_RANK", "0"))
        self.use_cuda_graph = os.environ.get("DRL_B200_CUDA_GRAPH", "0") == "1"
        self.sess = None
        self._kw = dict(num_action=num_action, input_shape=tuple(input_shape))
        self._main = self._target = None
        self._opt = None
        self._engine = None
        self._slot = 0
        self._last = {}
        self._lock = threading.RLock()   # actor threads sync from / act on this agent while the learner thread trains
        _AGENTS[model_name] = self

    # ---- engine management -----------------------------------------------------------
    def _ensure_init(self):
        if self._main is None:
            self._main = apex_value.init_params(**self._kw)
            self._target = apex_value.init_params(**self._kw)        # the two scopes are initialised independently
            z = np.zeros_like(self._main)
            self._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)

    def _pull_state(self):
        if self._engine is not None:
            self._main = self._engine.get_params(MAIN)
            self._target = self._engine.get_params(TARGET)
            self._opt = self._engine.get_opt_state()

    def _get_engine(self, batch):
        self._ensure_init()
        if self._engine is None or self._engine.B < batch:
            if self._engine is not None:
                self._pull_state()
                self._engine.close()
            self._engine = NativeApexLearner(
                batch=batch, num_action=self.num_action, input_shape=tuple(self.input_shape),
                discount_factor=self.discount_factor, gradient_clip_norm=self.gradient_clip_norm,
                reward_clipping=self.reward_clipping, start_learning_rate=self.start_learning_rate,
                end_learning_rate=self.end_learning_rate, learning_frame=self.learning_frame,
                device=self.device, num_slots=2, use_cuda_graph=self.use_cuda_graph)
            self._push_state()
        return self._engine

    def _push_state(self):
        e = self._engine
        e.set_params(self._main, MAIN)
        e.set_params(self._target, TARGET)
        o = self._opt
        e.set_opt_state(o["m"], o["v"], o["step"], o["beta1_power"], o["beta2_power"])

    # ---- reference API ---------------------------------------------------------------
    def target_to_main(self):
        """agent/apex.py:78-79: runs utils.main_to_target(main, target), i.e. target <- main."""
        self._ensure_init()
        if self._engine is not None:
            self._engine.target_to_main()
        else:
            self._target = self._main.copy()

    def _snapshot_params(self):
        with self._lock:
            self._ensure_init()
            if self._engine is not None:
                return self._engine.get_params(MAIN), self._engine.get_params(TARGET)
            return self._main.copy(), self._target.copy()

    def parameter_sync(self):
        """agent/apex.py:81-82 (utils.copy_src_to_dst(learner_name, model_name)): both scopes are trainable
        variables of the learner, so both are copied."""
        src = _AGENTS.get(self.learner_name)
        if src is None or src is self:
            return
        main, target = src._snapshot_params()            # trainable variables only, into caller-owned buffers
        with self._lock:
            self._ensure_init()
            self._main, self._target = main, target
            if self._engine is not None:
                self._engine.set_params(self._main, MAIN)
                self._engine.set_params(self._target, TARGET)

    def sync_policy(self, policy):
        """parameter_sync into a NativeApexPolicy (the actor side of ApexVectorActor): device to device from this
        agent's learner when it has one, otherwise from the host copy.  The actor only evaluates the main network, so
        only the main scope is copied."""
        with self._lock:
            if self._engine is not None:
                policy.sync_from(self._engine)
            else:
                self._ensure_init()
                policy.set_params(self._main)

    def set_session(self, sess):
        self.sess = sess
        self._main = None
        self._ensure_init()
        if self._engine is not None:
            self._push_state()

    def save_weights(self, path):
        self._ensure_init()
        self._pull_state()
        if not path.endswith(".npz"):
            path = path + ".npz"
        o = self._opt
        np.savez(path, main=self._main, target=self._target, m=o["m"], v=o["v"], step=np.int64(o["step"]),
                 beta1_power=np.float32(o["beta1_power"]), beta2_power=np.float32(o["beta2_power"]))

    def load_weights(self, path):
        if not path.endswith(".npz"):
            path = path + ".npz"
        z = np.load(path)
        n = apex_value.param_count(**self._kw)
        if z["main"].size != n:
            raise ValueError("checkpoint has %d parameters per scope, this agent has %d" % (z["main"].size, n))
        self._main, self._target = z["main"].astype(np.float32), z["target"].astype(np.float32)
        self._opt = dict(m=z["m"].astype(np.float32), v=z["v"].astype(np.float32), step=int(z["step"]),
                         beta1_power=float(z["beta1_power"]), beta2_power=float(z["beta2_power"]))
        if self._engine is not None:
            self._push_state()

    @staticmethod
    def _u8(state):
        st = np.asarray(state)
        if st.dtype != np.uint8:
            raise TypeError("states must be uint8 frames (the /255 normalisation runs on the GPU)")
        return st

    def get_policy_and_action(self, state, previous_action, epsilon):
        """agent/apex.py:88-102 -> (action, main_q_value, main_q_value[action])."""
        eng = self._engine if self._engine is not None else self._get_engine(1)
        q = eng.act(self._u8(state)[None], np.asarray([previous_action], np.int32))[0]
        if np.random.rand() > epsilon:
            action = np.argmax(q, axis=0)
        else:
            action = np.random.choice(self.num_action)
        return action, q, q[action]

    def get_td_error(self, state, next_state, previous_action, action, reward, done):
        """agent/apex.py:116-133 -> |target_value - state_action_value| [n]."""
        st = self._u8(np.stack(state))
        # evaluation only: reuse the training engine and go through it in chunks of its batch size; never rebuild it
        # for a larger n (train_apex.py calls this with `trajectory` transitions, which may exceed batch_size)
        eng = self._engine if self._engine is not None else self._get_engine(st.shape[0])
        out = np.empty(st.shape[0], np.float32)
        B = eng.B
        ns = self._u8(np.stack(next_state))
        for lo in range(0, st.shape[0], B):
            hi = min(lo + B, st.shape[0])
            out[lo:hi] = eng.td_error(st[lo:hi], ns[lo:hi], np.asarray(previous_action)[lo:hi],
                                      np.asarray(action)[lo:hi], np.asarray(reward)[lo:hi], np.asarray(done)[lo:hi])
        return out

    def _train(self, state, next_state, previous_action, action, reward, done, is_weight):
        st = self._u8(np.stack(state))
        if self._engine is not None and self._engine.B != st.shape[0]:
            self._pull_state()
            self._engine.close()
            self._engine = None
        eng = self._get_engine(st.shape[0])
        slot = self._slot
        self._slot = (self._slot + 1) % eng.num_slots
        eng.stage(slot, st, self._u8(np.stack(next_state)), previous_action, action, reward, done, is_weight)
        out, td = eng.step(slot)
        self._last = out
        return out["loss"], td

    def device_memory(self, capacity):
        """A prioritized replay memory of ``capacity`` transitions on this agent's GPU (buffer_queue.Memory's
        arithmetic); fill it with DeviceMemory.add, train from it with train_from_memory."""
        return DeviceMemory(self, capacity)

    def train_from_memory(self, memory, batch_size, u01=None):
        """One iteration of the learner loop's training half (train_apex.py:118-154) against a DeviceMemory:
        replay_buffer.sample(batch_size), the minibatch stack, distributed_train and the priority update, all on the GPU.
        ``u01`` ([batch_size] in [0, 1)) are the strata's uniforms; by default ``random.random()`` draws them exactly as
        Memory.sample does, so a host loop and a device loop seeded alike sample the same strata.  -> (loss, td_error)."""
        if dp.distributed():
            raise RuntimeError("train_from_memory: a DeviceMemory is local to one GPU; data-parallel training "
                               "(torch.distributed world > 1) uses Memory and distributed_train")
        if u01 is None:
            u01 = [random.random() for _ in range(batch_size)]
        if self._engine is not None and self._engine.B != batch_size:
            self._pull_state()
            self._engine.close()
            self._engine = None
        eng = self._get_engine(batch_size)
        slot = self._slot
        self._slot = (self._slot + 1) % eng.num_slots
        memory.replay.step_async(eng, slot, u01)
        out, td = eng.wait()
        self._last = out
        return out["loss"], td

    def distributed_train(self, state, next_state, previous_action, action, reward, done, is_weight):
        """agent/apex.py:135-154 -> (loss, td_error)."""
        return self._train(state, next_state, previous_action, action, reward, done, is_weight)

    def train(self, state, next_state, previous_action, action, reward, done):
        """agent/apex.py:156-168 (unit importance weights; returns None like the reference)."""
        self._train(state, next_state, previous_action, action, reward, done, None)

    learning_rate = property(lambda self: self._last.get("learning_rate"))
    grad_norm = property(lambda self: self._last.get("grad_norm"))
    value_loss = property(lambda self: self._last.get("loss"))
    num_env_frames = property(lambda self: self._last.get("step", (self._opt or {}).get("step", 0)))


class DeviceMemory:
    """The replay memory of train_apex.py:87 on the agent's GPU, for the device loop:

        memory = learner.device_memory(capacity)
        memory.add(state, next_state, previous_action, action, reward, done)   # get_td_error + the Memory.add loop
        loss, td_error = learner.train_from_memory(memory, batch_size)         # sample .. distributed_train .. update

    or, with the actors' ApexVectorActor pushing into an ApexDeviceFIFOQueue, ``memory.add_from_queue(queue)`` in place
    of the sample_batch(1) and the add.

    It outlives a rebuild of the agent's learner (another batch size): the agent passes its current learner to each
    call.  ``replay`` is the NativeApexReplay; ``n_entries``, ``beta``, ``total()`` and ``last_sample()`` read its state."""

    def __init__(self, agent, capacity):
        self.agent = agent
        self.capacity = int(capacity)
        self.replay = NativeApexReplay(self.capacity, device=agent.device, input_shape=tuple(agent.input_shape))

    def add(self, state, next_state, previous_action, action, reward, done):
        """learner.get_td_error(...) followed by replay_buffer.add(td_error[i], ...) for each transition in order
        (train_apex.py:99-116); the priorities are the learner's |td|, computed and applied on the device.  Transitions
        beyond the learner's batch go through in chunks of it, as get_td_error does."""
        a = self.agent
        st = a._u8(np.stack(state))
        ns = a._u8(np.stack(next_state))
        pa, ac = np.asarray(previous_action), np.asarray(action)
        rw, dn = np.asarray(reward), np.asarray(done)
        with a._lock:
            eng = a._engine if a._engine is not None else a._get_engine(st.shape[0])
            for lo in range(0, st.shape[0], eng.B):
                hi = min(lo + eng.B, st.shape[0])
                self.replay.add(eng, st[lo:hi], ns[lo:hi], pa[lo:hi], ac[lo:hi], rw[lo:hi], dn[lo:hi])

    def add_from_queue(self, queue, timeout_ms=-1):
        """``add`` of the oldest record of an ApexDeviceFIFOQueue (train_apex.py:94-116 without a host copy): the
        learner's |td| of its ``trajectory`` transitions and the store read the queue's GPU memory directly
        (trajectory <= the learner's batch).  Blocks while the queue is empty; ``timeout_ms`` >= 0 raises
        ``TimeoutError_`` with nothing changed.  One learner thread calls it, as it calls train_from_memory; actor
        threads may push into the queue and sync their policies from the agent meanwhile."""
        if dp.distributed():
            raise RuntimeError("add_from_queue: a DeviceMemory is local to one GPU; data-parallel training "
                               "(torch.distributed world > 1) uses Memory and distributed_train")
        a = self.agent
        with a._lock:
            eng = a._engine if a._engine is not None else a._get_engine(queue.trajectory)
        # the wait for a record runs without the agent's lock: actor threads take it in sync_policy meanwhile
        self.replay.add_from_queue(eng, queue, timeout_ms)

    n_entries = property(lambda self: self.replay.n_entries)
    beta = property(lambda self: self.replay.beta)

    def total(self):
        return self.replay.total()

    def last_sample(self):
        """(tree_index, priority, is_weight) of the most recent training step's draws."""
        return self.replay.last_sample()

    def close(self):
        self.replay.close()


def _locked(fn):
    def wrapper(self, *a, **k):
        with self._lock:
            return fn(self, *a, **k)
    wrapper.__name__, wrapper.__doc__ = fn.__name__, fn.__doc__
    return wrapper


# actor threads call these on a shared agent while the learner thread trains (in-process launch mode)
for _n in ('save_weights', 'load_weights', 'set_session', 'target_to_main', 'get_policy_and_action', 'get_td_error', '_train',
           'train_from_memory'):
    if hasattr(Agent, _n):
        setattr(Agent, _n, _locked(getattr(Agent, _n)))
