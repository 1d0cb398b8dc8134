"""H100-native stand-in for the reference's ``agent/r2d2.py``: same constructor kwargs, methods and return values, so
the learner branch of ``train_r2d2.py:87-165`` runs on it unchanged, with the TF1 graph replaced by ``drl_r2d2_*``.

  Agent.__init__       agent/r2d2.py:13-95
  Agent.get_td_error   agent/r2d2.py:97-130  (ONE sequence -> scalar)
  Agent.train          agent/r2d2.py:132-159 -> (loss, td_error [B])
  Agent.parameter_sync agent/r2d2.py:161-162 ; Agent.main_to_target :164-165 ; Agent.set_session :167-169
  Agent.get_action     agent/r2d2.py:171-191 -> (action, q_value[action], h', c')
  Agent.sync_policy    (new) parameter_sync into a NativeR2D2Policy (r2d2_policy.py), device to device from the learner
  Agent.train_calls    (new) read-only count of the training steps taken (train and train_from_memory); an
                       actor_server.R2D2PolicyServer syncs its policy whenever it has changed
  Agent.device_memory  (new) a DeviceMemory: the replay memory of train_r2d2.py:92-93 on the GPU (r2d2_replay.py);
                       DeviceMemory.add_from_queue ingests a batch of an R2D2DeviceFIFOQueue without a host copy
  Agent.train_from_memory (new) Memory.sample + the minibatch lists + train + Memory.update (train_r2d2.py:122-162)
                       as one device-resident step -> (loss, td_error)
  Agent.main_q_value_test / target_q_value_test   agent/r2d2.py:193-217
  Agent.save_weights / load_weights (new) both scopes and the Adam state in one .npz, as apex.Agent's
  Agent.set_n_step / set_priority_eta (new) the R2D2 paper's n-step targets and mixed max / mean priorities
                       (DESIGN.md section 22); switching keeps the parameters and the Adam state
"""
import os
import random
import threading

import numpy as np

from .. import dp
from ..model import r2d2_lstm
from ..r2d2_learner import MAIN, TARGET, NativeR2D2Learner
from ..r2d2_replay import NativeR2D2Replay

_AGENTS = {}


class Agent:

    def __init__(self, seq_len, burn_in, input_shape, num_action, lstm_size,
                 discount_factor, start_learning_rate, end_learning_rate,
                 learning_frame, gradient_clip_norm, model_name, learner_name):
        self.seq_len = seq_len
        self.burn_in = burn_in
        self.input_shape = list(input_shape)
        self.num_action = num_action
        self.lstm_size = lstm_size
        self.discount_factor = discount_factor
        self.start_learning_rate = start_learning_rate     # stored like the reference; its optimizer is a constant
        self.end_learning_rate = end_learning_rate         # AdamOptimizer(1e-4) without clipping (agent/r2d2.py:91-92)
        self.learning_frame = learning_frame
        self.model_name, self.learner_name = model_name, learner_name
        self.device = int(os.environ.get("LOCAL_RANK", "0"))
        self.use_cuda_graph = os.environ.get("DRL_B200_CUDA_GRAPH", "0") == "1"
        self.sess = None
        self._kw = dict(num_action=num_action, lstm_size=lstm_size, input_shape=tuple(input_shape))
        self._main = self._target = self._opt = None
        self._engine = None
        self._slot = 0
        self._last = {}
        self._train_calls = 0
        self.n_step, self.priority_eta = 1, None     # set_n_step / set_priority_eta
        self._lock = threading.RLock()   # actor threads sync from / act on this agent while the learner thread trains
        _AGENTS[model_name] = self

    def _ensure_init(self):
        if self._main is None:
            self._main = r2d2_lstm.init_params(**self._kw)
            self._target = r2d2_lstm.init_params(**self._kw)
            z = np.zeros_like(self._main)
            self._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)

    def _pull_state(self):
        if self._engine is not None:
            self._main, self._target = self._engine.get_params(MAIN), self._engine.get_params(TARGET)
            self._opt = self._engine.get_opt_state()

    def _push_state(self):
        e, o = self._engine, self._opt
        e.set_params(self._main, MAIN)
        e.set_params(self._target, TARGET)
        e.set_opt_state(o["m"], o["v"], o["step"], o["beta1_power"], o["beta2_power"])

    def _get_engine(self, batch):
        self._ensure_init()
        if self._engine is None or self._engine.B < batch:
            if self._engine is not None:
                self._pull_state()
                self._engine.close()
            self._engine = NativeR2D2Learner(
                batch=batch, seq_len=self.seq_len, burn_in=self.burn_in, num_action=self.num_action,
                lstm_size=self.lstm_size, input_shape=tuple(self.input_shape), discount_factor=self.discount_factor,
                device=self.device, num_slots=2, use_cuda_graph=self.use_cuda_graph, n_step=self.n_step,
                priority_eta=self.priority_eta)
            self._push_state()
        return self._engine

    def _rebuild_with(self, **kw):
        """Apply learner settings that live in the engine's configuration: the next call rebuilds the engine with
        the parameters, target network and Adam state it had."""
        with self._lock:
            if any(getattr(self, k) != v for k, v in kw.items()) and self._engine is not None:
                self._pull_state()
                self._engine.close()
                self._engine = None
            for k, v in kw.items():
                setattr(self, k, v)

    def set_n_step(self, n):
        """Train on n-step double-Q targets (the R2D2 paper uses n = 5; 1, the default, is the reference's one-step
        target).  The constructor keeps the reference's 12 arguments.  1 <= n <= seq_len - burn_in - 1."""
        n = int(n)
        if not 1 <= n <= self.seq_len - self.burn_in - 1:
            raise ValueError("n_step must be in [1, seq_len - burn_in - 1 = %d] (got %d)"
                             % (self.seq_len - self.burn_in - 1, n))
        self._rebuild_with(n_step=n)

    def set_priority_eta(self, eta):
        """Give each sequence the priority eta max_t |td| + (1 - eta) mean_t |td| (the R2D2 paper uses 0.9); None, the
        default, keeps the reference's |mean_t td|.  It applies to train's td_error, get_td_error and the priorities
        of a DeviceMemory."""
        if eta is not None:
            eta = float(eta)
            if not 0.0 <= eta <= 1.0:
                raise ValueError("priority_eta must be None or in [0, 1] (got %r)" % eta)
        self._rebuild_with(priority_eta=eta)

    @staticmethod
    def _u8(state):
        st = np.asarray(state)
        if st.dtype != np.uint8:
            raise TypeError("states must be uint8 frames (the /255 normalisation runs on the GPU)")
        return st

    def get_td_error(self, state, previous_action, action, h, c, reward, done):
        eng = self._get_engine(1)
        td = eng.td_error(self._u8(state)[None], np.asarray(previous_action)[None], np.asarray(action)[None],
                          np.asarray(h, np.float32)[None, 0], np.asarray(c, np.float32)[None, 0],
                          np.asarray(reward, np.float32)[None], np.asarray(done)[None])
        return float(td[0])

    def train(self, state, previous_action, action, h, c, reward, done, weight):
        st = self._u8(np.stack(state))
        if self._engine is not None and self._engine.B != st.shape[0]:
            self._pull_state()
            self._engine.close()
            self._engine = None
        eng = self._get_engine(st.shape[0])
        slot = self._slot
        self._slot = (self._slot + 1) % eng.num_slots
        eng.stage(slot, st, np.stack(previous_action), np.stack(action), np.stack(h)[:, 0], np.stack(c)[:, 0],
                  np.stack(reward), np.stack(done), weight)
        out, td = eng.step(slot)
        self._last = out
        self._train_calls += 1
        return out["loss"], td

    def device_memory(self, capacity):
        """A prioritized replay memory of ``capacity`` sequences on this agent's GPU (buffer_queue.Memory's
        arithmetic); fill it with DeviceMemory.add, train from it with train_from_memory."""
        return DeviceMemory(self, capacity)

    def train_from_memory(self, memory, batch_size, u01=None):
        """One iteration of the learner loop's training half (train_r2d2.py:122-162) against a DeviceMemory:
        per_replay_buffer.sample(batch_size), the minibatch lists, train and the priority update, all on the GPU.
        ``u01`` ([batch_size] in [0, 1)) are the strata's uniforms; by default ``random.random()`` draws them exactly as
        Memory.sample does, so a host loop and a device loop seeded alike sample the same strata.  -> (loss, td_error)."""
        if dp.distributed():
            raise RuntimeError("train_from_memory: a DeviceMemory is local to one GPU; data-parallel training "
                               "(torch.distributed world > 1) uses Memory and train")
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
        self._train_calls += 1
        return out["loss"], td

    def _snapshot_params(self):
        with self._lock:
            self._ensure_init()
            if self._engine is not None:
                return self._engine.get_params(MAIN), self._engine.get_params(TARGET)
            return self._main.copy(), self._target.copy()

    def parameter_sync(self):
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
        """parameter_sync into a NativeR2D2Policy (the actor side of R2D2VectorActor): device to device from this
        agent's learner when it has one, otherwise from the host copy of the main parameters."""
        with self._lock:
            if self._engine is not None:
                policy.sync_from(self._engine)
            else:
                self._ensure_init()
                policy.set_params(self._main)

    def main_to_target(self):
        self._ensure_init()
        if self._engine is not None:
            self._engine.main_to_target()
        else:
            self._target = self._main.copy()

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
        n = r2d2_lstm.param_count(**self._kw)
        if z["main"].size != n:
            raise ValueError("checkpoint has %d parameters per scope, this agent has %d (lstm_size %d)"
                             % (z["main"].size, n, self.lstm_size))
        self._main, self._target = z["main"].astype(np.float32), z["target"].astype(np.float32)
        self._opt = dict(m=z["m"].astype(np.float32), v=z["v"].astype(np.float32), step=int(z["step"]),
                         beta1_power=float(z["beta1_power"]), beta2_power=float(z["beta2_power"]))
        if self._engine is not None:
            self._push_state()

    def get_action(self, state, h, c, previous_action, epsilon):
        eng = self._engine if self._engine is not None else self._get_engine(1)
        q, h2, c2 = eng.act(self._u8(state)[None], np.asarray([previous_action], np.int32),
                            np.asarray(h, np.float32)[None], np.asarray(c, np.float32)[None])
        q = q[0]
        if np.random.rand() > epsilon:
            action = np.argmax(q)
        else:
            action = np.random.choice(self.num_action)
        return action, q[action], h2[0], c2[0]

    def _unroll_q(self, key, state, h, c, done, previous_action):
        eng = self._get_engine(1)
        S = self.seq_len
        eng.td_error(self._u8(np.stack(state))[None], np.asarray(previous_action)[None], np.zeros((1, S), np.int32),
                     np.asarray(h, np.float32)[None, 0], np.asarray(c, np.float32)[None, 0], np.zeros((1, S), np.float32),
                     np.asarray(done)[None])
        return eng.taps(1)[key][0]

    def main_q_value_test(self, state, h, c, done, previous_action):
        return self._unroll_q("main_q", state, h, c, done, previous_action)

    def target_q_value_test(self, state, h, c, done, previous_action):
        return self._unroll_q("target_q", state, h, c, done, previous_action)

    @property
    def train_calls(self):
        """Training steps taken so far: calls of train and train_from_memory that returned."""
        return self._train_calls

    value_loss = property(lambda self: self._last.get("loss"))
    grad_norm = property(lambda self: self._last.get("grad_norm"))


class DeviceMemory:
    """The replay memory of train_r2d2.py:92-93 on the agent's GPU, for the device loop:

        memory = learner.device_memory(capacity)
        q = r2d2_queue.sample_batch()
        memory.add(q.state, q.previous_action, q.action, q.previous_h, q.previous_c, q.reward, q.done)
        loss, td_error = learner.train_from_memory(memory, batch_size)  # sample .. train .. update

    or, with the actors' R2D2VectorActor recording into an R2D2DeviceFIFOQueue, ``memory.add_from_queue(queue)`` in
    place of the sample_batch and the add.

    It outlives a rebuild of the agent's learner (another batch size): the agent passes its current learner to each
    call.  ``replay`` is the NativeR2D2Replay; ``n_entries``, ``beta``, ``total()`` and ``last_sample()`` read its state."""

    def __init__(self, agent, capacity):
        self.agent = agent
        self.capacity = int(capacity)
        self.replay = NativeR2D2Replay(self.capacity, seq_len=agent.seq_len, num_action=agent.num_action,
                                       input_shape=tuple(agent.input_shape), device=agent.device,
                                       lstm_size=agent.lstm_size)

    @staticmethod
    def _step0(x):
        """h / c as stored by the actors ([n, S, L]) or already at step 0 ([n, L]) -> [n, L] float32."""
        x = np.asarray(x, np.float32)
        return x[:, 0] if x.ndim == 3 else x

    def add(self, state, previous_action, action, h, c, reward, done):
        """learner.get_td_error(...) followed by per_replay_buffer.add(td_error, ...) for each sequence of one
        R2D2FIFOQueue.sample_batch() in order (train_r2d2.py:101-120); the priorities are the learner's |td|, computed
        for the whole batch at once and applied on the device.  Sequences beyond the learner's batch go through in
        chunks of it."""
        a = self.agent
        st = a._u8(state)
        pa, ac = np.asarray(previous_action), np.asarray(action)
        h0, c0 = self._step0(h), self._step0(c)
        rw, dn = np.asarray(reward), np.asarray(done)
        with a._lock:
            eng = a._engine if a._engine is not None else a._get_engine(st.shape[0])
            for lo in range(0, st.shape[0], eng.B):
                hi = min(lo + eng.B, st.shape[0])
                self.replay.add(eng, st[lo:hi], pa[lo:hi], ac[lo:hi], h0[lo:hi], c0[lo:hi], rw[lo:hi], dn[lo:hi])

    def add_from_queue(self, queue, timeout_ms=-1):
        """``add`` of the oldest ``queue.batch_size`` sequences of an R2D2DeviceFIFOQueue (train_r2d2.py:97-120
        without a host copy): the learner's |td| of the batch and the store read the queue's GPU memory directly.
        Blocks while fewer than a batch are queued; ``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing
        changed.  One learner thread calls it, as it calls train_from_memory; actor threads may record into the
        queue and sync their policies from the agent meanwhile."""
        if dp.distributed():
            raise RuntimeError("add_from_queue: a DeviceMemory is local to one GPU; data-parallel training "
                               "(torch.distributed world > 1) uses Memory and train")
        a = self.agent
        with a._lock:
            eng = a._engine if a._engine is not None else a._get_engine(queue.batch_size)
        # the wait for a full batch runs without the agent's lock: actor threads take it in sync_policy meanwhile
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
for _n in ('save_weights', 'load_weights', 'set_session', 'main_to_target', 'get_action', 'get_td_error', 'train', 'main_q_value_test', 'target_q_value_test',
           'train_from_memory'):
    if hasattr(Agent, _n):
        setattr(Agent, _n, _locked(getattr(Agent, _n)))
