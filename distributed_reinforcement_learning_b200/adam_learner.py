"""The part of the Ape-X, A3C and R2D2 wrappers that is the same for all three: the main / target parameters, the TF1
Adam state and the data-parallel step with grad_scale = 1 / world (dp.py), on top of ``LearnerHandle``."""
import ctypes as C

import numpy as np

from . import _native as N
from . import dp
from .learner_handle import LearnerHandle

MAIN, TARGET = 0, 1


class AdamLearnerHandle(LearnerHandle):
    # ---- parameters / optimizer state -------------------------------------------------
    def set_params(self, flat, which=MAIN):
        a = N.as_c(flat, np.float32, (self.param_count,), "params")
        N.check(self._fn("set_params")(self._h, int(which), N.ptr(a), a.size))

    def get_params(self, which=MAIN):
        a = np.empty(self.param_count, np.float32)
        N.check(self._fn("get_params")(self._h, int(which), N.ptr(a), a.size))
        return a

    def set_opt_state(self, m, v, step, beta1_power=0.9, beta2_power=0.999):
        am = N.as_c(m, np.float32, (self.param_count,), "m")
        av = N.as_c(v, np.float32, (self.param_count,), "v")
        N.check(self._fn("set_opt_state")(self._h, N.ptr(am), N.ptr(av), am.size, int(step), float(beta1_power),
                                          float(beta2_power)))

    def get_opt_state(self):
        m = np.empty(self.param_count, np.float32)
        v = np.empty(self.param_count, np.float32)
        st, b1, b2 = C.c_int64(), C.c_float(), C.c_float()
        N.check(self._fn("get_opt_state")(self._h, N.ptr(m), N.ptr(v), m.size, C.byref(st), C.byref(b1),
                                          C.byref(b2)))
        return dict(m=m, v=v, step=int(st.value), beta1_power=float(b1.value), beta2_power=float(b2.value))

    # ---- step ----------------------------------------------------------------------------
    def step(self, slot=0):
        """-> what wait() returns.  With torch.distributed initialised (world > 1) the step is data parallel (dp.py)."""
        self.step_async(slot)
        return self.wait()

    def step_async(self, slot=0):
        if dp.distributed():
            self._dp.step_async(slot)           # data parallel: see dp.py
        else:
            N.check(self._fn("step_async")(self._h, slot))
