"""R2D2 learner bench leg (BASELINE.json configs[4]; `python bench.py --workload r2d2`): frames/s of
``r2d2.Agent.train`` on synthetic sequences -- B=16 sequences (config.json:94) of seq_len=80 with burn_in=40 (the sizes
BASELINE.json names; the reference ships 15/7), 84x84x1 frames, LSTM 64, 4 actions, one H100.

  value : device-resident (two staged slots alternate, the whole step is one CUDA graph)
  e2e   : through the C-ABI with HOST buffers (per-step H2D of the sequences, host reads loss + B priorities)
  roofline : dominant contraction kernel vs the measured bf16 peak; the two recurrence kernels are reported beside it
  cpu_baseline : the float32 torch-CPU oracle (oracle/r2d2_torch.py), a restatement of the TF1 reference
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

A, L, C = 4, 64, 1
# BASELINE.json names seq_len 80 / burn_in 40; DRL_R2D2_SEQ / DRL_R2D2_BURN select another shape (the reference ships 15 / 7)
B, S, BI = 16, int(os.environ.get("DRL_R2D2_SEQ", "80")), int(os.environ.get("DRL_R2D2_BURN", "40"))
METRIC = "R2D2 learner frames/sec (B=16,seq_len=%d,burn_in=%d,84x84x1,LSTM 64)" % (S, BI)


def kernel_flops(name, M):
    n = name[7:] if name.startswith("target_") else name
    tbl = {"conv1_fwd": 2.0 * M * 400 * 32 * 64 * C, "conv2_fwd": 2.0 * M * 81 * 64 * 512,
           "conv3_fwd": 2.0 * M * 49 * 64 * 576, "lstm_x_fwd": 2.0 * M * 256 * 3392,
           "lstm_wgrad": 2.0 * 3456 * 256 * M, "lstm_dgrad": 2.0 * M * 3392 * 256,
           "conv3_wgrad": 2.0 * M * 49 * 64 * 576, "conv3_dgrad": 2.0 * M * 49 * 64 * 576,
           "conv2_wgrad": 2.0 * M * 81 * 64 * 512, "conv2_dgrad": 2.0 * M * 81 * 64 * 512,
           "conv1_wgrad": 2.0 * M * 400 * 32 * 64 * C}
    return tbl.get(n)


def cpu_reference(steps, warmup, cores, b=B, s=S, bi=BI):
    import torch
    from oracle import r2d2_torch as rt
    torch.set_num_threads(cores)
    d = rt.make_sequences(b, S=s, A=A)
    args = [d[k] for k in rt.TRAIN_FIELDS]
    Lr = rt.Learner(dtype=torch.float32, seq_len=s, burn_in=bi)
    for _ in range(warmup):
        Lr.train(*args)
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        Lr.train(*args)
        ts.append(time.perf_counter() - t0)
    sec = float(np.sum(ts)) / max(len(ts), 1)
    return dict(value=b * s / sec, unit="frames/s", cores=cores, kind="port", ms_per_step=sec * 1e3,
                sample="%d timed steps (+%d warm-up) of the float32 torch-CPU restatement of r2d2.Agent.train (2 x %d "
                       "recurrent network steps, autograd BPTT, TF1 Adam) at B=%d" % (steps, warmup, s, b))


def run(args, bench):
    if args.impl == "reference":
        steps, warm = max(1, min(args.steps, 10)), max(1, min(args.warmup, 2))
        cb = cpu_reference(steps, warm, bench.usable_cores())
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": cb["value"], "unit": "frames/s", "n_gpus": 1,
                          "steps": steps, "warmup": warm, "ms_per_step": cb["ms_per_step"], "higher_is_better": True,
                          "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                          "config": {"workload": "R2D2 learner step (BASELINE configs[4]), CPU torch restatement of the "
                                                 "TF1 reference", "global_batch": B, "seq_len": S, "burn_in": BI},
                          "cpu_baseline": cb, "gpu_launches": 0,
                          "e2e": {"value": cb["value"], "unit": "frames/s", "h2d_bytes_per_step": 0,
                                  "d2h_bytes_per_step": 0}}))
        return
    import torch
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("the R2D2 bench leg is single-GPU")
    torch.cuda.set_device(0)
    K, W = args.steps, max(args.warmup, 3)
    use_graph = not args.no_graph
    mode = 2 if args.math_mode > 2 else args.math_mode
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=BI, num_action=A, lstm_size=L, input_shape=(84, 84, C),
                            use_cuda_graph=use_graph, math_mode=mode)
    eng.set_params(r2d2_lstm.init_params(seed=0, num_action=A, input_shape=(84, 84, C)), MAIN)
    eng.set_params(r2d2_lstm.init_params(seed=1, num_action=A, input_shape=(84, 84, C)), TARGET)
    rng = np.random.default_rng(11)
    keep, hb = [], []

    def pinned(shape, dtype):
        t = torch.empty(int(np.prod(shape)) * np.dtype(dtype).itemsize, dtype=torch.uint8).pin_memory()
        keep.append(t)
        return t.numpy().view(dtype).reshape(shape)
    for i in range(3):
        gens = (((B, S, 84, 84, C), np.uint8, lambda s: rng.integers(0, 256, s, dtype=np.uint8)),
                ((B, S), np.int32, lambda s: rng.integers(0, A, s).astype(np.int32)),
                ((B, S), np.int32, lambda s: rng.integers(0, A, s).astype(np.int32)),
                ((B, L), np.float32, lambda s: np.clip(rng.standard_normal(s) * 0.5, -0.999, 0.999).astype(np.float32)),
                ((B, L), np.float32, lambda s: rng.standard_normal(s).astype(np.float32)),
                ((B, S), np.float32, lambda s: rng.standard_normal(s).astype(np.float32)),
                ((B, S), np.uint8, lambda s: (rng.random(s) < 0.02).astype(np.uint8)),
                ((B,), np.float32, lambda s: rng.uniform(0.2, 1.0, s).astype(np.float32)))
        arrs = []
        for shape, dt, gen in gens:
            a = pinned(shape, dt)
            a[...] = gen(shape)
            arrs.append(a)
        hb.append(arrs)
    h2d = int(sum(a.nbytes for a in hb[0]))
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
        eng.step_async(i % 2)
    e1.record(ext)
    eng.wait()
    torch.cuda.synchronize()
    dev_ms = e0.elapsed_time(e1)
    clocks = sampler.stop()
    launches = eng.launches_per_step() * K
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
    M = B * S
    name, kms = next(((n, ms) for n, ms in top if kernel_flops(n, M)), top[0])
    fl = kernel_flops(name, M)
    ach = fl / (kms * 1e-3) / 1e12 if fl else 0.0
    line = {"metric": METRIC, "value": M / (dev_ms / K * 1e-3), "unit": "frames/s", "n_gpus": 1, "steps": K, "warmup": W,
            "ms_per_step": dev_ms / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": {"workload": "R2D2 learner step (BASELINE configs[4]): B=16 sequences x seq_len %d (burn_in %d), "
                                   "84x84x1 uint8, A=4, LSTM 64, stored-state unroll of main and target scope, BPTT, TF1 Adam" % (S, BI),
                       "global_batch": B, "seq_len": S, "burn_in": BI, "cuda_graph": bool(use_graph),
                       "math_mode": bench.MATH_MODES[mode],
                       "l2": "activations + workspace ~0.9 GB/step > 126 MB L2; two staged slots alternate",
                       "timing": "CUDA events on the learner's compute stream around K back-to-back steps"},
            "e2e": {"value": M / (ms_e2e / K * 1e-3), "unit": "frames/s", "h2d_bytes_per_step": h2d,
                    "d2h_bytes_per_step": 32 + 4 * B, "ms_per_step": ms_e2e / K,
                    "path": "pinned host arrays -> drl_r2d2_stage (copy stream) -> drl_r2d2_step_async -> drl_r2d2_wait"},
            "gpu_launches": launches, "clocks": clocks,
            "roofline": {"kernel": name, "bound": "tensor", "achieved": ach, "peak": peaks["tf_sus"], "unit": "TFLOP/s",
                         "frac": ach / peaks["tf_sus"], "frac_of_3xtf32_ceiling": ach / (peaks["tf_sus"] / 6.0),
                         "traffic": None, "kernel_ms": kms, "share_of_step": kms / tot,
                         "peak_source": peaks["src"] + " bf16 sustained"},
            "recurrence_ms": {n: ms for n, ms in prof if "unroll" in n},
            "kernels_ms": [[n, round(ms, 4)] for n, ms in top], "step_ms_sum_of_kernels": tot,
            "last_step": {k: out[k] for k in ("loss", "grad_norm", "step")}}
    if args.cpu_baseline:
        line["cpu_baseline"] = cpu_reference(2, 1, bench.usable_cores())
    eng.close()
    print(json.dumps(line))
