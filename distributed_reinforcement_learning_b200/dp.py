"""Data-parallel plumbing shared by the learners: one process per GPU, every rank feeds its own minibatch, ONE
``all_reduce(SUM)`` of the gradient bucket (loss scalars in its tail) between the two halves of the step
(``drl_<family>_forward_backward`` / ``drl_<family>_apply``).  The Ape-X, A3C and R2D2 losses are batch MEANS, so their
update of the undivided global batch is the summed bucket times 1 / world_size (``grad_scale``); the IMPALA losses are
batch sums, so its apply takes the summed bucket as it is (learner.py)."""
import ctypes as C

from . import _native as N


def distributed():
    try:
        import torch.distributed as dist
    except Exception:      # pragma: no cover
        return False
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


class BucketAllReduce:
    def __init__(self, family, handle, device):
        self.family, self._h, self.device = family, handle, int(device)
        self._bucket = self._stream = None

    def _fn(self, name):
        return getattr(N.lib, "drl_%s_%s" % (self.family, name))

    def _tensor(self):
        """torch view (no copy) of the device gradient bucket [padded grads | loss sums | pad]."""
        if self._bucket is None:
            import torch
            p, n, s = C.c_void_p(), C.c_int64(), C.c_void_p()
            N.check(self._fn("grad_bucket")(self._h, C.byref(p), C.byref(n)))
            N.check(self._fn("stream")(self._h, C.byref(s)))

            class _View:
                __cuda_array_interface__ = {"shape": (int(n.value),), "typestr": "<f4", "data": (int(p.value), False),
                                            "version": 2}
            dev = "cuda:%d" % self.device
            self._bucket = torch.as_tensor(_View(), device=dev)
            self._stream = torch.cuda.ExternalStream(int(s.value or 0), device=dev)
        return self._bucket

    def all_reduce(self):
        """all_reduce(SUM) of the bucket on the learner's stream: after the backward pass, before the update."""
        import torch
        import torch.distributed as dist
        t = self._tensor()
        with torch.cuda.stream(self._stream):
            dist.all_reduce(t, op=dist.ReduceOp.SUM)

    def step_async(self, slot):
        """forward+backward -> all_reduce(SUM) on the learner's stream -> clip + Adam with grad_scale = 1 / world."""
        import torch.distributed as dist
        N.check(self._fn("forward_backward")(self._h, slot))
        self.all_reduce()
        N.check(self._fn("apply")(self._h, C.c_float(1.0 / dist.get_world_size())))
