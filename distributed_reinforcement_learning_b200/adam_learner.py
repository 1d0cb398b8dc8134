"""The part of the Ape-X, A3C and R2D2 wrappers that is the same for all three: each drives one ``drl_<family>_*``
learner handle of the C-ABI (include/drl_b200.h), and these entry points differ only in that prefix."""
import ctypes as C

import numpy as np

from . import _native as N
from . import dp

MAIN, TARGET = 0, 1


class AdamLearnerHandle:
    family = None      # "apex", "a3c" or "r2d2": the C-ABI prefix

    def _fn(self, name):
        return getattr(N.lib, "drl_%s_%s" % (self.family, name))

    def _create(self, cfg, device, num_slots):
        self._h = C.c_void_p()
        N.check(self._fn("create")(C.byref(cfg), C.byref(self._h)))
        n = C.c_int64()
        N.check(self._fn("param_count")(self._h, C.byref(n)))
        self.param_count = int(n.value)
        self.num_slots = int(num_slots)
        self._keep = [None] * self.num_slots      # the staged host arrays stay alive until the slot is restaged
        self._dp = dp.BucketAllReduce(self.family, self._h, int(device))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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

    def get_grads(self):
        a = np.empty(self.param_count, np.float32)
        N.check(self._fn("get_grads")(self._h, N.ptr(a), a.size))
        return a

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

    # ---- introspection ---------------------------------------------------------------------
    def read_buffer(self, name, count):
        a = np.empty(int(count), np.float32)
        N.check(self._fn("read_buffer")(self._h, name.encode(), N.ptr(a), a.size))
        return a

    def profile_step(self, slot=0, max_kernels=128):
        names = C.create_string_buffer(8192)
        ms = np.zeros(max_kernels, np.float32)
        cnt = C.c_int32()
        N.check(self._fn("profile_step")(self._h, slot, names, len(names), N.ptr(ms), max_kernels, C.byref(cnt)))
        nm = names.value.decode().split("\n") if cnt.value else []
        return list(zip(nm, [float(x) for x in ms[:cnt.value]]))

    def last_step_ms(self):
        ms = C.c_float()
        N.check(self._fn("last_step_ms")(self._h, C.byref(ms)))
        return float(ms.value)

    def launches_per_step(self):
        n = C.c_int32()
        N.check(self._fn("launches_per_step")(self._h, C.byref(n)))
        return int(n.value)

    def stream_ptr(self):
        s = C.c_void_p()
        N.check(self._fn("stream")(self._h, C.byref(s)))
        return int(s.value or 0)
