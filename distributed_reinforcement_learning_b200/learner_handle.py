"""The part of the IMPALA, Ape-X, A3C and R2D2 learner wrappers that is the same for all four: each drives one
``drl_<family>_*`` learner handle of the C-ABI (include/drl_b200.h), and these entry points differ only in that
prefix."""
import ctypes as C

import numpy as np

from . import _native as N
from . import dp


class LearnerHandle:
    family = None      # "learner" (IMPALA), "apex", "a3c" or "r2d2": the C-ABI prefix

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

    def get_grads(self):
        a = np.empty(self.param_count, np.float32)
        N.check(self._fn("get_grads")(self._h, N.ptr(a), a.size))
        return a

    # ---- introspection ---------------------------------------------------------------------
    def read_buffer(self, name, count):
        a = np.empty(int(count), np.float32)
        N.check(self._fn("read_buffer")(self._h, name.encode(), N.ptr(a), a.size))
        return a

    def profile_step(self, slot=0, max_kernels=128):
        """One real step with a CUDA event before every launch -> [(kernel name, device ms)]."""
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
