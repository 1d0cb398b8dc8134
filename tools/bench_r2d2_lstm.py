"""R2D2 learner step at LSTM widths 64, 256 and 512 (the paper's network is 512 wide): B = 16 sequences of seq_len 80
with burn-in 40, 84x84x1 frames, 4 actions, CUDA graphs, two staged slots alternating, math mode 2.

At 64 the recurrence runs one CTA per sequence (r2d2_lstm_fwd_kernel); at 256 and 512 it runs on a thread-block
cluster of L / 32 CTAs (csrc/r2d2_cluster.cuh).  The sizes are timed in alternating blocks of K back-to-back steps
(CUDA events on each learner's compute stream), so the spread between blocks shows beside the difference between
sizes.  Then one profiled step per size gives the per-kernel times.  Prints the card's name, power limit and maximum SM
clock (read in the same run), then one JSON line per size.

    python tools/bench_r2d2_lstm.py [--steps 20] [--warmup 5] [--rounds 5] [--sizes 64,256,512]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

B, S, BI, A, C = 16, 80, 40, 4, 1
KERNELS = ("lstm_unroll_fwd", "target_lstm_unroll_fwd", "lstm_unroll_bwd", "lstm_x_fwd", "target_lstm_x_fwd",
           "lstm_wgrad", "lstm_dgrad")


def gpu_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        info.update(smi_name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:        # the timing does not depend on it; say what is missing
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def make_learner(L, rng):
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=BI, num_action=A, lstm_size=L, input_shape=(84, 84, C),
                            use_cuda_graph=True, math_mode=2)
    kw = dict(num_action=A, lstm_size=L, input_shape=(84, 84, C))
    eng.set_params(r2d2_lstm.init_params(seed=0, **kw), MAIN)
    eng.set_params(r2d2_lstm.init_params(seed=1, **kw), TARGET)
    for slot in range(2):
        eng.stage(slot, rng.integers(0, 256, (B, S, 84, 84, C), dtype=np.uint8),
                  rng.integers(0, A, (B, S)).astype(np.int32), rng.integers(0, A, (B, S)).astype(np.int32),
                  np.clip(rng.standard_normal((B, L)) * 0.5, -0.999, 0.999).astype(np.float32),
                  rng.standard_normal((B, L)).astype(np.float32), rng.standard_normal((B, S)).astype(np.float32),
                  (rng.random((B, S)) < 0.02).astype(np.uint8), rng.uniform(0.2, 1.0, B).astype(np.float32))
    return eng


def time_block(eng, K):
    import torch
    ext = torch.cuda.ExternalStream(eng.stream_ptr(), device="cuda:0")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(ext)
    for i in range(K):
        eng.step_async(i % 2)
    e1.record(ext)
    out, _ = eng.wait()
    torch.cuda.synchronize()
    if not np.isfinite(out["loss"]):
        raise RuntimeError("non-finite loss")
    return e0.elapsed_time(e1) / K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", default="64,256,512")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_r2d2_lstm needs a CUDA device")
    torch.cuda.set_device(0)
    sizes = [int(x) for x in args.sizes.split(",")]
    info = gpu_info()
    print(json.dumps({"gpu": info}))
    rng = np.random.default_rng(11)
    engs = {L: make_learner(L, rng) for L in sizes}
    try:
        for L in sizes:
            for i in range(max(args.warmup, 3)):
                engs[L].step(i % 2)
        ms = {L: [] for L in sizes}
        for _ in range(args.rounds):
            for L in sizes:
                ms[L].append(time_block(engs[L], args.steps))
        for L in sizes:
            eng = engs[L]
            prof = [eng.profile_step(0) for _ in range(3)][-1]
            kern = {}
            for n, t in prof:
                if n in KERNELS:
                    kern[n] = round(kern.get(n, 0.0) + t, 4)
            med = float(np.median(ms[L]))
            print(json.dumps({
                "lstm_size": L, "recurrence": "one CTA per sequence" if L == 64 else "cluster of %d CTAs" % (L // 32),
                "ms_per_step": round(med, 4), "ms_per_step_blocks": [round(x, 4) for x in ms[L]],
                "frames_per_s": round(B * S / (med * 1e-3), 1), "launches_per_step": eng.launches_per_step(),
                "clusters": dict(zip(("size", "max_fwd", "max_bwd"), eng.recurrence_clusters())),
                "kernels_ms": kern, "profiled_step_ms": round(sum(t for _, t in prof), 4),
                "config": {"batch": B, "seq_len": S, "burn_in": BI, "frames": "84x84x%d" % C, "num_action": A,
                           "cuda_graph": True, "math_mode": 2, "steps_per_block": args.steps, "rounds": args.rounds,
                           "timing": "CUDA events on the compute stream around K back-to-back steps, sizes alternating"},
                "gpu": info}))
    finally:
        for eng in engs.values():
            eng.close()


if __name__ == "__main__":
    main()
