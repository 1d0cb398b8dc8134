"""H100-native stand-in for the reference's ``agent/impala.py``: same constructor kwargs, same
methods, same return values -- so the learner branch of ``train_impala.py:89-113`` runs on it
unchanged -- with the TF1 graph + ``tf.Session`` replaced by the CUDA learner behind the C-ABI.

  Agent.__init__            agent/impala.py:11-103   (graph construction -> records the config)
  Agent.set_session         agent/impala.py:114-116  (also initialises all variables, like the reference)
  Agent.train               agent/impala.py:132-148  -> stage + one fused device step
  Agent.train_from_queue    (new) the same step on a batch of a DeviceFIFOQueue, staged device to device
  Agent.get_policy_and_action  agent/impala.py:118-130
  Agent.parameter_sync      agent/impala.py:111-112  (learner -> this agent's variables)
  Agent.sync_policy         (new) parameter_sync into a NativePolicy (policy.py), device to device from the learner
  Agent.save_weights / load_weights   agent/impala.py:105-109

The graph attributes the reference exposes (``vs``, ``clipped_rho``, ``vs_plus_1``, ``pg_advantage``,
``pi_loss``, ``baseline_loss``, ``entropy``, ``total_loss``, ``learning_rate``, ``num_env_frames``;
agent/impala.py:68-96) are exposed as the values of the most recent ``train`` call.

Data parallelism (new; SURVEY.md section 8(e)): launched under torchrun with ``torch.distributed``
initialised, every rank feeds its own shard of the global batch to ``train`` and the gradient
bucket is all-reduced (SUM) over NCCL before the identical replicated update.
"""
import os
import threading

import numpy as np

from .. import dp
from ..learner import NativeLearner
from ..model import impala_actor_critic

_AGENTS = {}          # model_name -> Agent, the stand-in for TF variable scopes in one process


class Agent:

    def __init__(self, trajectory, input_shape, num_action, lstm_hidden_size,
                 discount_factor, start_learning_rate, end_learning_rate,
                 learning_frame, baseline_loss_coef, entropy_coef,
                 gradient_clip_norm, reward_clipping, model_name, learner_name):
        if reward_clipping not in ("abs_one", "soft_asymmetric"):          # utils.py:45
            raise AssertionError("reward_clipping must be 'abs_one' or 'soft_asymmetric'")
        self.input_shape = list(input_shape)
        self.trajectory = trajectory
        self.num_action = num_action
        self.lstm_hidden_size = lstm_hidden_size
        self.discount_factor = discount_factor
        self.start_learning_rate = start_learning_rate
        self.end_learning_rate = end_learning_rate
        self.learning_frame = learning_frame
        self.baseline_loss_coef = baseline_loss_coef
        self.entropy_coef = entropy_coef
        self.gradient_clip_norm = gradient_clip_norm
        self.reward_clipping = reward_clipping
        self.model_name = model_name
        self.learner_name = learner_name
        self.recurrent = False         # set_recurrent
        self.device = int(os.environ.get("LOCAL_RANK", "0"))
        # the whole step is one CUDA graph by default (the benchmarked path); DRL_B200_CUDA_GRAPH=0 launches eagerly
        self.use_cuda_graph = os.environ.get("DRL_B200_CUDA_GRAPH", "1") != "0"
        # actor threads call parameter_sync()/get_policy_and_action() while the learner thread trains (in-process mode
        # of train_impala.py): every method that touches the agent's state or its engine holds this lock
        self._lock = threading.RLock()
        self.sess = None
        self._kw = dict(num_action=num_action, lstm_hidden_size=lstm_hidden_size, input_shape=tuple(input_shape))
        self._params = None            # flat float32 (host copy, authoritative while no engine exists)
        self._ms = None
        self._step = 0
        self._engine = None
        self._last = {}
        self._slot = 0
        _AGENTS[model_name] = self

    # ---- engine management -----------------------------------------------------------
    def _ensure_init(self):
        if self._params is None:
            self._params = impala_actor_critic.init_params(**self._kw)
            self._ms = np.ones_like(self._params)      # TF1 RMSProp slot initial value
            self._step = 0

    def _pull_state(self):
        if self._engine is not None:
            self._params = self._engine.get_params()
            self._ms, self._step = self._engine.get_opt_state()

    def _get_engine(self, batch):
        self._ensure_init()
        if self._engine is None or self._engine.B != batch:
            if self._engine is not None:
                self._pull_state()
                self._engine.close()
            self._engine = NativeLearner(
                batch=batch, trajectory=self.trajectory, num_action=self.num_action,
                lstm_hidden_size=self.lstm_hidden_size, input_shape=tuple(self.input_shape),
                discount_factor=self.discount_factor, start_learning_rate=self.start_learning_rate,
                end_learning_rate=self.end_learning_rate, learning_frame=self.learning_frame,
                baseline_loss_coef=self.baseline_loss_coef, entropy_coef=self.entropy_coef,
                gradient_clip_norm=self.gradient_clip_norm, reward_clipping=self.reward_clipping,
                device=self.device, num_slots=2, use_cuda_graph=self.use_cuda_graph, recurrent=self.recurrent)
            self._engine.set_params(self._params)
            self._engine.set_opt_state(self._ms, self._step)
        return self._engine

    def set_recurrent(self, recurrent=True):
        """Choose how ``train`` / ``train_from_queue`` treat the LSTM (the constructor keeps the reference's 14
        arguments).  False (the default) trains as the reference does: one LSTM step from each step's recorded (h, c).
        True unrolls the LSTM through each trajectory with BPTT, restarting from the recorded state after every done
        (NativeLearner(recurrent=True), DESIGN.md section 21).  Parameters, RMSProp state and checkpoints are the same in
        both modes: switching keeps them and rebuilds the learner engine at the next step."""
        with self._lock:
            recurrent = bool(recurrent)
            if recurrent != self.recurrent and self._engine is not None:
                self._pull_state()
                self._engine.close()
                self._engine = None
            self.recurrent = recurrent

    # ---- reference API ---------------------------------------------------------------
    def save_weights(self, path):
        """tf.train.Saver().save: parameters + RMSProp slots + global_step, TF layouts, one .npz."""
        with self._lock:
            self._ensure_init()
            self._pull_state()
            if not path.endswith(".npz"):
                path = path + ".npz"
            np.savez(path, params=self._params, ms=self._ms, step=np.int64(self._step))

    def load_weights(self, path):
        with self._lock:
            if not path.endswith(".npz"):
                path = path + ".npz"
            z = np.load(path)
            n = impala_actor_critic.param_count(**self._kw)
            if z["params"].size != n:
                raise ValueError("checkpoint has %d parameters, this agent has %d" % (z["params"].size, n))
            self._params = z["params"].astype(np.float32)
            self._ms = z["ms"].astype(np.float32)
            self._step = int(z["step"])
            if self._engine is not None:
                self._engine.set_params(self._params)
                self._engine.set_opt_state(self._ms, self._step)

    def _snapshot_params(self):
        """Parameters only, into a buffer the CALLER owns (no rebinding of this agent's fields from a foreign thread)."""
        with self._lock:
            self._ensure_init()
            return self._engine.get_params() if self._engine is not None else self._params.copy()

    def parameter_sync(self):
        """Copy the learner's variables into this agent (utils.copy_src_to_dst, utils.py:6-22): trainable variables
        only -- the RMSProp slots are not part of the copy."""
        src = _AGENTS.get(self.learner_name)
        if src is None or src is self:
            return
        params = src._snapshot_params()
        with self._lock:
            self._params = params
            if self._ms is None:
                self._ms = np.ones_like(self._params)
            if self._engine is not None:
                self._engine.set_params(self._params)

    def sync_policy(self, policy):
        """parameter_sync into a NativePolicy (the actor side of VectorActor): device to device from this agent's
        learner when it has one, otherwise from the host copy of the parameters."""
        with self._lock:
            if self._engine is not None:
                policy.sync_from(self._engine)
            else:
                self._ensure_init()
                policy.set_params(self._params)

    def set_session(self, sess):
        """Stores the session object (unused) and (re-)initialises every variable, as
        ``sess.run(tf.global_variables_initializer())`` does (agent/impala.py:114-116)."""
        with self._lock:
            self.sess = sess
            self._params = None
            self._ensure_init()
            if self._engine is not None:
                self._engine.set_params(self._params)
                self._engine.set_opt_state(self._ms, self._step)

    def get_policy_and_action(self, state, previous_action, h, c):
        """agent/impala.py:118-130 -> (action, policy, max(policy), h', c')."""
        with self._lock:
            eng = self._engine if self._engine is not None else self._get_engine(1)
            st = np.asarray(state)
            if st.dtype != np.uint8:
                st = np.clip(np.rint(st), 0, 255).astype(np.uint8)
            policy, rh, rc = eng.act(st[None], np.asarray([previous_action], np.int32),
                                     np.asarray(h, np.float32)[None], np.asarray(c, np.float32)[None])
            policy, rh, rc = policy[0], rh[0], rc[0]
            p = policy.astype(np.float64)
            action = np.random.choice(self.num_action, p=p / p.sum())
            return action, policy, max(policy), rh, rc

    def train(self, state, reward, action, done, behavior_policy, previous_action, initial_h, initial_c):
        """agent/impala.py:132-148 -> (pi_loss, value_loss, entropy, learning_rate).
        ``state`` is the raw uint8 [B, T, 84, 84, 4] batch; the /255 of :133 happens on the device."""
        with self._lock:
            state = np.asarray(state)
            if state.dtype != np.uint8:
                raise TypeError("state must be uint8 frames (the /255 normalisation runs on the GPU)")
            eng = self._get_engine(state.shape[0])
            slot = self._slot
            self._slot = (self._slot + 1) % eng.num_slots
            eng.stage(slot, state, reward, action, done, behavior_policy, previous_action, initial_h, initial_c)
            out = eng.step(slot)
            self._last = out
            return out["pi_loss"], out["baseline_loss"], out["entropy"], out["learning_rate"]

    def train_from_queue(self, queue, timeout_ms=-1):
        """``train`` on the oldest batch of a ``DeviceFIFOQueue`` (the actors' recorders fill it on the GPU): the
        batch is staged device to device, then the same step runs.  Blocks until the queue holds a batch
        (``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing changed).  -> (pi_loss, value_loss, entropy,
        learning_rate), as ``train``.  One learner thread calls it; do not interleave it with ``train`` from another
        thread (with two staging slots, a ``train`` that runs while this call waits for a batch can reuse its slot)."""
        with self._lock:
            if dp.distributed():
                raise RuntimeError("train_from_queue is single-replica: the queue lives on one device")
            eng = self._get_engine(queue.batch_size)
            slot = self._slot
            self._slot = (slot + 1) % eng.num_slots    # taken now, so a train() meanwhile picks the other slot
        # wait for the batch without the agent's lock: actor threads sync their policies from this agent meanwhile
        try:
            eng.stage_from_queue(slot, queue, timeout_ms)
        except Exception:
            with self._lock:
                if self._slot == (slot + 1) % eng.num_slots:
                    self._slot = slot                  # nothing was staged: the slot is not used up
            raise
        with self._lock:
            out = eng.step(slot)
            self._last = out
            return out["pi_loss"], out["baseline_loss"], out["entropy"], out["learning_rate"]

    # ---- graph attributes as last-step values (agent/impala.py:68-96) -----------------
    def _tap(self, name):
        if self._engine is None:
            raise RuntimeError("no train() call has run yet")
        return self._engine.taps()[name]

    vs = property(lambda self: self._tap("vs"))
    clipped_rho = property(lambda self: self._tap("clipped_rho"))
    vs_plus_1 = property(lambda self: self._tap("vs_plus_1"))
    pg_advantage = property(lambda self: self._tap("pg_advantage"))
    pi_loss = property(lambda self: self._last.get("pi_loss"))
    baseline_loss = property(lambda self: self._last.get("baseline_loss"))
    entropy = property(lambda self: self._last.get("entropy"))
    total_loss = property(lambda self: self._last.get("total_loss"))
    learning_rate = property(lambda self: self._last.get("learning_rate"))
    grad_norm = property(lambda self: self._last.get("grad_norm"))
    num_env_frames = property(lambda self: self._last.get("step", self._step))
