"""A3C learner bench leg (`python bench.py --workload a3c`): transitions/s of ``a3c.Agent.train`` on one unroll of
trajectory = 32 synthetic 84x84x4 transitions (config.json:2-41), one H100.  Same structure as tools/bench_apex.py."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

A, B = 4, 32
METRIC = "A3C learner transitions/sec (B=32,84x84x4,A=4)"


def cpu_reference(steps, warmup, cores):
    import torch
    from oracle import a3c_torch as at
    torch.set_num_threads(cores)
    b = at.make_transitions(B, A=A)
    args = [b[k] for k in at.TRAIN_FIELDS]
    L = at.Learner(dtype=torch.float32, num_action=A)
    for _ in range(warmup):
        L.train(*args)
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        L.train(*args)
        ts.append(time.perf_counter() - t0)
    sec = float(np.sum(ts)) / max(len(ts), 1)
    return dict(value=B / sec, unit="transitions/s", cores=cores, kind="port", ms_per_step=sec * 1e3,
                sample="%d timed steps (+%d warm-up) of the float32 torch-CPU restatement of a3c.Agent.train at B=%d"
                       % (steps, warmup, B))


def run(args, bench):
    if args.impl == "reference":
        steps, warm = max(1, min(args.steps, 50)), max(1, min(args.warmup, 3))
        cb = cpu_reference(steps, warm, bench.usable_cores())
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": cb["value"], "unit": "transitions/s", "n_gpus": 1,
                          "steps": steps, "warmup": warm, "ms_per_step": cb["ms_per_step"], "higher_is_better": True,
                          "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                          "config": {"workload": "A3C learner step, CPU torch restatement of the TF1 reference",
                                     "global_batch": B}, "cpu_baseline": cb, "gpu_launches": 0,
                          "e2e": {"value": cb["value"], "unit": "transitions/s", "h2d_bytes_per_step": 0,
                                  "d2h_bytes_per_step": 0}}))
        return
    import ctypes as C
    import torch
    import bench_apex
    from distributed_reinforcement_learning_b200 import _native as N
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.model import actor_critic
    torch.cuda.set_device(0)
    K, W = args.steps, max(args.warmup, 3)
    use_graph = not args.no_graph
    mode = 2 if args.math_mode > 2 else args.math_mode
    eng = NativeA3CLearner(batch=B, num_action=A, use_cuda_graph=use_graph, math_mode=mode)
    eng.set_params(actor_critic.init_params(seed=0, num_action=A))
    rng = np.random.default_rng(7)
    keep, hb = [], []
    for i in range(3):
        arrs = []
        for shape, dt, gen in (((B, 84, 84, 4), np.uint8, lambda s: rng.integers(0, 256, s, dtype=np.uint8)),
                               ((B, 84, 84, 4), np.uint8, lambda s: rng.integers(0, 256, s, dtype=np.uint8)),
                               ((B,), np.int32, lambda s: rng.integers(0, A, s).astype(np.int32)),
                               ((B,), np.int32, lambda s: rng.integers(0, A, s).astype(np.int32)),
                               ((B,), np.float32, lambda s: rng.standard_normal(s).astype(np.float32)),
                               ((B,), np.uint8, lambda s: (rng.random(s) < 0.1).astype(np.uint8))):
            t = torch.empty(int(np.prod(shape)) * np.dtype(dt).itemsize, dtype=torch.uint8).pin_memory()
            a = t.numpy().view(dt).reshape(shape)
            a[...] = gen(shape)
            keep.append(t)
            arrs.append(a)
        hb.append(arrs)
    h2d = int(sum(a.nbytes for a in hb[0]))
    s_ptr = C.c_void_p()
    N.check(N.lib.drl_a3c_stream(eng._h, C.byref(s_ptr)))
    ext = torch.cuda.ExternalStream(int(s_ptr.value), device="cuda:0")
    eng.stage(0, *hb[0])
    eng.stage(1, *hb[1])
    for i in range(W):
        eng.step(i % 2)
    sampler = bench.ClockSampler(0)
    torch.cuda.synchronize()
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for i in range(K):
        N.check(N.lib.drl_a3c_step_async(eng._h, i % 2))
    e1.record(ext)
    o = N.A3cOut()
    N.check(N.lib.drl_a3c_wait(eng._h, C.byref(o)))
    torch.cuda.synchronize()
    dev_ms = e0.elapsed_time(e1)
    clocks = sampler.stop()
    n = C.c_int32()
    N.check(N.lib.drl_a3c_launches_per_step(eng._h, C.byref(n)))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    eng.stage(0, *hb[0])
    for i in range(K):
        N.check(N.lib.drl_a3c_step_async(eng._h, i % 2))
        if i + 1 < K:
            eng.stage((i + 1) % 2, *hb[(i + 1) % 3])
        N.check(N.lib.drl_a3c_wait(eng._h, C.byref(o)))
    torch.cuda.synchronize()
    ms_e2e = (time.perf_counter() - t0) * 1e3
    peaks = bench.measured_peaks()
    eng.stage(0, *hb[0])
    names = C.create_string_buffer(8192)
    ms = np.zeros(128, np.float32)
    cnt = C.c_int32()
    for _ in range(3):
        N.check(N.lib.drl_a3c_profile_step(eng._h, 0, names, len(names), N.ptr(ms), 128, C.byref(cnt)))
    prof = list(zip(names.value.decode().split("\n"), [float(x) for x in ms[:cnt.value]]))
    tot = sum(v for _, v in prof)
    top = sorted(prof, key=lambda kv: -kv[1])
    name, kms = next(((k, v) for k, v in top if bench_apex.kernel_flops(k, B)), top[0])
    fl = bench_apex.kernel_flops(name, B)
    ach = fl / (kms * 1e-3) / 1e12 if fl else 0.0
    line = {"metric": METRIC, "value": B / (dev_ms / K * 1e-3), "unit": "transitions/s", "n_gpus": 1, "steps": K,
            "warmup": W, "ms_per_step": dev_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": "A3C learner step: one unroll of 32 transitions, 84x84x4 uint8 state+next_state, A=4, "
                                   "A2C losses, TF1 Adam", "global_batch": B, "cuda_graph": bool(use_graph),
                       "math_mode": bench.MATH_MODES[mode], "l2": "working set < L2; two staged slots alternate"},
            "e2e": {"value": B / (ms_e2e / K * 1e-3), "unit": "transitions/s", "h2d_bytes_per_step": h2d,
                    "d2h_bytes_per_step": 32, "ms_per_step": ms_e2e / K},
            "gpu_launches": int(n.value) * K, "clocks": clocks,
            "roofline": {"kernel": name, "bound": "tensor", "achieved": ach, "peak": peaks["tf_sus"], "unit": "TFLOP/s",
                         "frac": ach / peaks["tf_sus"], "traffic": None, "kernel_ms": kms, "share_of_step": kms / tot},
            "kernels_ms": [[k, round(v, 4)] for k, v in top],
            "last_step": {"pi_loss": o.pi_loss, "baseline_loss": o.baseline_loss, "entropy": o.entropy, "step": o.step}}
    if args.cpu_baseline:
        line["cpu_baseline"] = cpu_reference(5, 1, bench.usable_cores())
    eng.close()
    print(json.dumps(line))
