"""H100-native stand-in for the reference's ``agent/a3c.py``: same constructor kwargs, methods and return values (the
learner branch of ``train_a3c.py`` runs on it unchanged), with the TF1 graph replaced by ``drl_a3c_*``.

  Agent.__init__               agent/a3c.py:11-83
  Agent.train                  agent/a3c.py:85-103 -> (pi_loss, value_loss, entropy, learning_rate)
  Agent.train_from_queue       train on the oldest record of an A3CDeviceFIFOQueue, staged device to device
  Agent.set_session            agent/a3c.py:105-107
  Agent.get_policy_and_action  agent/a3c.py:109-119 -> (action, policy, max_prob)
  Agent.parameter_sync         agent/a3c.py:121-122
  Agent.sync_policy            parameter_sync into a NativeA3CPolicy (actor.py: A3CVectorActor)
"""
import os
import threading

import numpy as np

from .. import dp
from ..a3c_learner import NativeA3CLearner
from ..model import actor_critic

_AGENTS = {}


class Agent:

    def __init__(self, input_shape, num_action, discount_factor,
                 start_learning_rate, end_learning_rate,
                 learning_frame, baseline_loss_coef, entropy_coef,
                 gradient_clip_norm, reward_clipping, model_name, learner_name):
        if reward_clipping not in ("abs_one", "soft_asymmetric"):
            raise AssertionError("reward_clipping must be 'abs_one' or 'soft_asymmetric'")
        self.input_shape = list(input_shape)
        self.num_action = num_action
        self._cfg = dict(discount_factor=discount_factor, start_learning_rate=start_learning_rate,
                         end_learning_rate=end_learning_rate, learning_frame=learning_frame,
                         baseline_loss_coef=baseline_loss_coef, entropy_coef=entropy_coef,
                         gradient_clip_norm=gradient_clip_norm, reward_clipping=reward_clipping)
        self.model_name, self.learner_name = model_name, learner_name
        self.device = int(os.environ.get("LOCAL_RANK", "0"))
        self.use_cuda_graph = os.environ.get("DRL_B200_CUDA_GRAPH", "0") == "1"
        self.sess = None
        self._kw = dict(num_action=num_action, input_shape=tuple(input_shape))
        self._params = self._opt = None
        self._engine = None
        self._slot = 0
        self._last = {}
        self._lock = threading.RLock()   # actor threads sync from / act on this agent while the learner thread trains
        _AGENTS[model_name] = self

    def _ensure_init(self):
        if self._params is None:
            self._params = actor_critic.init_params(**self._kw)
            z = np.zeros_like(self._params)
            self._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)

    def _pull_state(self):
        if self._engine is not None:
            self._params = self._engine.get_params()
            self._opt = self._engine.get_opt_state()

    def _get_engine(self, batch):
        self._ensure_init()
        if self._engine is None or self._engine.B < batch:
            if self._engine is not None:
                self._pull_state()
                self._engine.close()
            self._engine = NativeA3CLearner(batch=batch, num_action=self.num_action, input_shape=tuple(self.input_shape),
                                            device=self.device, num_slots=2, use_cuda_graph=self.use_cuda_graph,
                                            **self._cfg)
            self._engine.set_params(self._params)
            o = self._opt
            self._engine.set_opt_state(o["m"], o["v"], o["step"], o["beta1_power"], o["beta2_power"])
        return self._engine

    @staticmethod
    def _u8(state):
        st = np.asarray(state)
        if st.dtype != np.uint8:
            raise TypeError("states must be uint8 frames (the /255 normalisation runs on the GPU)")
        return st

    def train(self, state, next_state, previous_action, action, reward, done):
        st = self._u8(np.stack(state))
        if self._engine is not None and self._engine.B != st.shape[0]:
            self._pull_state()
            self._engine.close()
            self._engine = None
        eng = self._get_engine(st.shape[0])
        slot = self._slot
        self._slot = (self._slot + 1) % eng.num_slots
        eng.stage(slot, st, self._u8(np.stack(next_state)), previous_action, action, reward, done)
        out = eng.step(slot)
        self._last = out
        return out["pi_loss"], out["baseline_loss"], out["entropy"], out["learning_rate"]

    def train_from_queue(self, queue, timeout_ms=-1):
        """``train`` on the oldest record of an ``A3CDeviceFIFOQueue`` (the actors' recorders fill it on the GPU): the
        record is staged device to device, then the same step runs.  Blocks until the queue holds a record
        (``timeout_ms`` >= 0 raises ``TimeoutError_`` with nothing changed).  -> (pi_loss, value_loss, entropy,
        learning_rate), as ``train``.  One learner thread calls it; do not interleave it with ``train`` from another
        thread."""
        with self._lock:
            if dp.distributed():
                raise RuntimeError("train_from_queue is single-replica: the queue lives on one device")
            if self._engine is not None and self._engine.B != queue.trajectory:
                self._pull_state()
                self._engine.close()
                self._engine = None
            eng = self._get_engine(queue.trajectory)
            slot = self._slot
            self._slot = (slot + 1) % eng.num_slots    # taken now, so a train() meanwhile picks the other slot
        # wait for the record without the agent's lock: actor threads sync their policies from this agent meanwhile
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

    def set_session(self, sess):
        self.sess = sess
        self._params = None
        self._ensure_init()
        if self._engine is not None:
            self._engine.set_params(self._params)
            o = self._opt
            self._engine.set_opt_state(o["m"], o["v"], o["step"], o["beta1_power"], o["beta2_power"])

    def get_policy_and_action(self, state, previous_action):
        eng = self._engine if self._engine is not None else self._get_engine(1)
        policy = eng.act(self._u8(state)[None], np.asarray([previous_action], np.int32))[0][0]
        p = policy.astype(np.float64)
        action = np.random.choice(self.num_action, p=p / p.sum())
        return action, policy, policy[action]

    def parameter_sync(self):
        src = _AGENTS.get(self.learner_name)
        if src is None or src is self:
            return
        src._ensure_init()
        src._pull_state()
        self._params = src._params.copy()
        if self._opt is None:
            z = np.zeros_like(self._params)
            self._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
        if self._engine is not None:
            self._engine.set_params(self._params)

    def sync_policy(self, policy):
        """parameter_sync into a NativeA3CPolicy (the actor side of A3CVectorActor): device to device from this
        agent's learner when it has one, otherwise from the host copy of the parameters."""
        with self._lock:
            if self._engine is not None:
                policy.sync_from(self._engine)
            else:
                self._ensure_init()
                policy.set_params(self._params)

    learning_rate = property(lambda self: self._last.get("learning_rate"))
    grad_norm = property(lambda self: self._last.get("grad_norm"))
    num_env_frames = property(lambda self: self._last.get("step", (self._opt or {}).get("step", 0)))


def _locked(fn):
    def wrapper(self, *a, **k):
        with self._lock:
            return fn(self, *a, **k)
    wrapper.__name__, wrapper.__doc__ = fn.__name__, fn.__doc__
    return wrapper


# actor threads call these on a shared agent while the learner thread trains (in-process launch mode); a sync from an
# actor thread never meets the learner thread's engine rebuild in train
for _n in ('train', 'set_session', 'get_policy_and_action', 'parameter_sync'):
    setattr(Agent, _n, _locked(getattr(Agent, _n)))
