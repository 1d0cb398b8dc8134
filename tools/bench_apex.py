"""Ape-X learner bench leg (BASELINE.json configs[3]; `python bench.py --workload apex`): transitions/s of
``apex.Agent.distributed_train`` on synthetic 84x84x4 minibatches, B=32 (config.json:154), one H100.

  value : device-resident (two staged slots alternate, the whole step is one CUDA graph)
  e2e   : through the C-ABI with HOST buffers: every step copies that step's minibatch (2 x B frames + scalars) from
          pinned memory and reads back the loss and the B new priorities |td|
  roofline : dominant contraction kernel (per-launch CUDA-event time from drl_apex_profile_step) vs the measured bf16 peak
  cpu_baseline : the float32 torch-CPU oracle (oracle/apex_torch.py), a restatement of the TF1 reference
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

A = 4
METRIC = "Ape-X learner transitions/sec (B=32,84x84x4,A=4)"


def kernel_flops(name, B):
    tgt = name.startswith("target_")
    n = name[7:] if tgt else name
    M = B if tgt else 2 * B           # forward rows: main [s ; s'], target [s']
    tbl = {"conv1_fwd": 2.0 * M * 400 * 32 * 256, "conv2_fwd": 2.0 * M * 81 * 64 * 512,
           "conv3_fwd": 2.0 * M * 49 * 64 * 576, "heads_l1_fwd": 2.0 * M * 512 * 3392,
           "heads_l2_fwd": 4.0 * M * 256 * 256,
           "heads_l1_wgrad": 2.0 * 3392 * 512 * B, "heads_l1_dgrad": 2.0 * B * 3392 * 512,
           "heads_l2_wgrad": 4.0 * B * 256 * 256, "heads_l2_dgrad": 4.0 * B * 256 * 256,
           "conv3_wgrad": 2.0 * B * 49 * 64 * 576, "conv3_dgrad": 2.0 * B * 49 * 64 * 576,
           "conv2_wgrad": 2.0 * B * 81 * 64 * 512, "conv2_dgrad": 2.0 * B * 81 * 64 * 512,
           "conv1_wgrad": 2.0 * B * 400 * 32 * 256}
    return tbl.get(n)


def step_flops(B):
    fwd = 7738112 + 2 * 3392 * 256 + 2 * 256 * 256 + 256 * (A + 1)     # MAC per row: convs + two streams
    return 2.0 * fwd * (3 * B) + 2.0 * 2.0 * fwd * B


def cpu_reference(steps, warmup, B, cores):
    import torch
    from oracle import apex_torch as ax
    torch.set_num_threads(cores)
    b = ax.make_transitions(B, A=A)
    args = [b[k] for k in ax.TRAIN_FIELDS]
    L = ax.Learner(dtype=torch.float32, num_action=A)
    for _ in range(warmup):
        L.distributed_train(*args)
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        L.distributed_train(*args)
        ts.append(time.perf_counter() - t0)
    sec = float(np.sum(ts)) / max(len(ts), 1)
    return dict(value=B / sec, unit="transitions/s", cores=cores, kind="port", ms_per_step=sec * 1e3,
                sample="%d timed steps (+%d warm-up) of the float32 torch-CPU restatement of apex.Agent.distributed_train "
                       "(3 dueling-network evaluations, autograd, clip 40, TF1 Adam) at B=%d" % (steps, warmup, B))


def run(args, bench):
    B = 32
    if args.impl == "reference":
        steps, warm = max(1, min(args.steps, 50)), max(1, min(args.warmup, 3))
        cb = cpu_reference(steps, warm, B, bench.usable_cores())
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": cb["value"], "unit": "transitions/s",
                          "n_gpus": 1, "steps": steps, "warmup": warm, "ms_per_step": cb["ms_per_step"],
                          "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
                          "data": "synthetic", "config": {"workload": "Ape-X learner step (BASELINE configs[3]), CPU "
                                                          "torch restatement of the TF1 reference", "global_batch": B},
                          "cpu_baseline": cb, "gpu_launches": 0,
                          "e2e": {"value": cb["value"], "unit": "transitions/s", "h2d_bytes_per_step": 0,
                                  "d2h_bytes_per_step": 0}}))
        return
    import torch
    from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET, NativeApexLearner
    from distributed_reinforcement_learning_b200.model import apex_value
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("the Ape-X bench leg is single-GPU (value_loss is a batch MEAN; see DESIGN.md)")
    torch.cuda.set_device(0)
    K, W = args.steps, max(args.warmup, 3)
    use_graph = not args.no_graph
    mode = 2 if args.math_mode > 2 else args.math_mode
    eng = NativeApexLearner(batch=B, num_action=A, use_cuda_graph=use_graph, math_mode=mode)
    eng.set_params(apex_value.init_params(seed=0, num_action=A), MAIN)
    eng.set_params(apex_value.init_params(seed=1, num_action=A), TARGET)
    rng = np.random.default_rng(7)

    def pinned(shape, dtype):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        t = torch.empty(n, dtype=torch.uint8).pin_memory()
        return t, t.numpy().view(dtype).reshape(shape)
    keep, hb = [], []
    for i in range(3):
        arrs = []
        for shape, dt, gen in (((B, 84, 84, 4), np.uint8, lambda s: rng.integers(0, 256, s, dtype=np.uint8)),
                               ((B, 84, 84, 4), np.uint8, lambda s: rng.integers(0, 256, s, dtype=np.uint8)),
                               ((B,), np.int32, lambda s: rng.integers(0, A, s).astype(np.int32)),
                               ((B,), np.int32, lambda s: rng.integers(0, A, s).astype(np.int32)),
                               ((B,), np.float32, lambda s: rng.standard_normal(s).astype(np.float32)),
                               ((B,), np.uint8, lambda s: (rng.random(s) < 0.1).astype(np.uint8)),
                               ((B,), np.float32, lambda s: rng.uniform(0.2, 1.0, s).astype(np.float32))):
            t, a = pinned(shape, dt)
            a[...] = gen(shape)
            keep.append(t)
            arrs.append(a)
        hb.append(arrs)
    h2d = int(sum(a.nbytes for a in hb[0]))

    # device-resident
    eng.stage(0, *hb[0])
    eng.stage(1, *hb[1])
    for i in range(W):
        eng.step(i % 2)
    ext = torch.cuda.ExternalStream(eng.stream_ptr(), device="cuda:0")
    sampler = bench.ClockSampler(0)
    torch.cuda.synchronize()
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(K):
        eng.step_async(i % 2)                   # K whole steps back to back on the learner's compute stream
    e1.record(ext)
    eng.wait()
    torch.cuda.synchronize()
    dev_ms = e0.elapsed_time(e1)
    clocks = sampler.stop()
    launches = eng.launches_per_step() * K

    # end to end: H2D of the step's minibatch + step + the host reads loss and td_error
    for i in range(2):
        eng.stage(i % 2, *hb[i % 3])
        eng.step(i % 2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.stage(0, *hb[0])
    for i in range(K):
        eng.step_async(i % 2)
        if i + 1 < K:
            eng.stage((i + 1) % 2, *hb[(i + 1) % 3])
        out, td = eng.wait()
    torch.cuda.synchronize()
    ms_e2e = (time.perf_counter() - t0) * 1e3

    peaks = bench.measured_peaks()
    eng.stage(0, *hb[0])
    prof = [eng.profile_step(0) for _ in range(3)][-1]
    tot = sum(ms for _, ms in prof)
    top = sorted(prof, key=lambda kv: -kv[1])
    name, kms = next(((n, ms) for n, ms in top if kernel_flops(n, B)), top[0])
    fl = kernel_flops(name, B)
    ach = fl / (kms * 1e-3) / 1e12 if fl else 0.0
    line = {"metric": METRIC, "value": B / (dev_ms / K * 1e-3), "unit": "transitions/s", "n_gpus": 1, "steps": K,
            "warmup": W, "ms_per_step": dev_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": "Ape-X DQN learner step (BASELINE configs[3]): B=32 transitions, 84x84x4 uint8 "
                                   "state+next_state, A=4, dueling double-DQN, TF1 Adam; glorot random-init parameters",
                       "global_batch": B, "cuda_graph": bool(use_graph), "math_mode": bench.MATH_MODES[mode],
                       "l2": "working set ~60 MB < 126 MB L2: two staged slots alternate, latency-bound step",
                       "timing": "CUDA events on the learner's compute stream around K back-to-back steps"},
            "e2e": {"value": B / (ms_e2e / K * 1e-3), "unit": "transitions/s", "h2d_bytes_per_step": h2d,
                    "d2h_bytes_per_step": 32 + 4 * B, "ms_per_step": ms_e2e / K,
                    "path": "pinned host arrays -> drl_apex_stage (copy stream, overlaps the previous step) -> "
                            "drl_apex_step_async -> drl_apex_wait (loss + B priorities read on the host every step)"},
            "gpu_launches": launches, "clocks": clocks,
            "roofline": {"kernel": name, "bound": "tensor", "achieved": ach, "peak": peaks["tf_sus"], "unit": "TFLOP/s",
                         "frac": ach / peaks["tf_sus"], "traffic": None, "kernel_ms": kms, "share_of_step": kms / tot,
                         "peak_source": peaks["src"] + " bf16 sustained",
                         "note": "B=32 is a latency-bound step (96 forward / 32 backward images): small grids, see DESIGN.md"},
            "kernels_ms": [[n, round(ms, 4)] for n, ms in top], "step_ms_sum_of_kernels": tot,
            "step_tflops": step_flops(B) / (dev_ms / K * 1e-3) / 1e12,
            "last_step": {k: out[k] for k in ("loss", "grad_norm", "step")}}
    if args.cpu_baseline:
        line["cpu_baseline"] = cpu_reference(5, 1, B, bench.usable_cores())
    eng.close()
    print(json.dumps(line))
