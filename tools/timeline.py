"""True kernel timeline of one learner step inside the CUDA-graph replay (both streams).

    python tools/timeline.py [--math-mode 2] [--no-graph]

Arms drl_debug_trace: CTA 0 of every kernel records {globaltimer, grid, block} when it starts.
Prints the start times relative to the first kernel, the gap to the next start on the device
and the launch geometry, so each kernel can be recognised (conv1_fwd = 2000 CTAs x 160 threads, ...)."""
import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributed_reinforcement_learning_b200 import _native as N   # noqa: E402
from distributed_reinforcement_learning_b200.learner import NativeLearner   # noqa: E402
from bench import synth_batch   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--math-mode", type=int, default=2)
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--collective", choices=["peer", "nccl"], default="peer", help="under torchrun (N > 1)")
    ap.add_argument("--back-to-back", action="store_true",
                    help="enqueue all steps without host synchronisation (steady state) and print the last one")
    a = ap.parse_args()
    B, T = a.batch, 20
    world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    eng = NativeLearner(batch=B, trajectory=T, num_action=18, use_cuda_graph=not a.no_graph, math_mode=a.math_mode,
                        device=local)
    if world > 1 and a.collective == "peer":
        eng.enable_peer_exchange()
    bt = synth_batch(B, 1)
    fields = ("state", "reward", "action", "done", "behavior_policy", "previous_action", "initial_h", "initial_c")
    for s in range(2):
        eng.stage(s, *[bt[f] for f in fields])
    for i in range(6):
        eng.step(i % 2)
    buf = torch.zeros(8001, dtype=torch.int64, device="cuda")
    N.check(N.lib.drl_debug_trace(C.c_void_p(buf.data_ptr())))
    per_step = []
    if a.back_to_back:
        nsteps = max(a.steps, 6)
        buf.zero_()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()
        for i in range(nsteps):
            eng.step_async(i % 2)
        eng.wait()
        torch.cuda.synchronize()
        h = buf.cpu().numpy()
        n = int(h[0])
        rec = sorted((int(h[1 + 2 * j]), int(h[2 + 2 * j])) for j in range(n))
        per = n // nsteps
        per_step = [rec[k * per:(k + 1) * per] for k in range(nsteps)]
        print("# back-to-back: step periods (first kernel to first kernel, us): %s" % ", ".join(
            "%.1f" % ((per_step[k + 1][0][0] - per_step[k][0][0]) / 1e3) for k in range(nsteps - 1)))
        per_step = per_step[:-1] if False else per_step
    for i in range(0 if a.back_to_back else a.steps):
        buf.zero_()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()
        eng.step(i % 2)
        torch.cuda.synchronize()
        h = buf.cpu().numpy()
        n = int(h[0])
        rec = sorted((int(h[1 + 2 * j]), int(h[2 + 2 * j])) for j in range(n))
        per_step.append(rec)
    N.check(N.lib.drl_debug_trace(C.c_void_p(0)))
    if world > 1:
        dist.barrier()
        eng.close()
        dist.barrier()
        dist.destroy_process_group()
        if rank != 0:
            return
    rec = per_step[-1]
    t0 = rec[0][0]
    print("# %d kernels, first start -> last start %.1f us (steps: %s)" % (
        len(rec), (rec[-1][0] - t0) / 1e3, ", ".join("%.1f" % ((r[-1][0] - r[0][0]) / 1e3) for r in per_step)))
    print("# start_us  next_start_in_us  grid  block")
    for j, (t, g) in enumerate(rec):
        nxt = (rec[j + 1][0] - t) / 1e3 if j + 1 < len(rec) else 0.0
        print("%9.1f %9.1f %7d %5d" % ((t - t0) / 1e3, nxt, g >> 32, g & 0xffffffff))


if __name__ == "__main__":
    main()
