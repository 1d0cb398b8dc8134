"""IMPALA learner step in its two modes: stored-state (the reference's: one LSTM step from each step's recorded state)
and recurrent (the LSTM unrolled through the trajectory with BPTT, DESIGN.md section 21).  B = 32 trajectories of T = 20,
84x84x4 frames, A = 18, math mode 5, CUDA graphs, a device-resident batch (both staged slots filled once, then stepped
alternately).

The two modes are timed in alternating blocks of K back-to-back steps (CUDA events on each learner's compute stream), so
the spread between blocks shows beside the difference between modes.  Then one profiled step per mode gives the
recurrence and BPTT kernel times.  Prints the card's name, power limit and maximum SM clock (read in the same run), then
one JSON line per mode.

    python tools/bench_impala_recurrent.py [--steps 20] [--warmup 5] [--rounds 7]
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

B, T, A = 32, 20, 18
KERNELS = ("lstm_fwd", "lstm_x_reduce", "lstm_gates_fwd", "lstm_unroll_fwd", "lstm_gates_bwd", "lstm_unroll_bwd",
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


def make_learner(recurrent, batch, params):
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    eng = NativeLearner(batch=B, trajectory=T, num_action=A, use_cuda_graph=True, math_mode=5, recurrent=recurrent)
    eng.set_params(params)
    from oracle import synthetic
    for slot in range(2):
        eng.stage(slot, *[batch[k] for k in synthetic.TRAIN_FIELDS])
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
    out = eng.wait()
    torch.cuda.synchronize()
    if not np.isfinite(out["total_loss"]):
        raise RuntimeError("non-finite loss")
    return e0.elapsed_time(e1) / K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_impala_recurrent needs a CUDA device")
    torch.cuda.set_device(0)
    from oracle import impala_torch as it
    from oracle import synthetic
    info = gpu_info()
    print(json.dumps({"gpu": info}))
    batch = synthetic.make_batch(B, T=T, A=A, seed=5)
    params = it.flatten_params(it.init_params(0, torch.float32, num_action=A))
    modes = {"stored_state": False, "recurrent": True}
    engs = {m: make_learner(r, batch, params) for m, r in modes.items()}
    try:
        for m in modes:
            for i in range(max(args.warmup, 3)):
                engs[m].step(i % 2)
        ms = {m: [] for m in modes}
        for _ in range(args.rounds):
            for m in modes:
                ms[m].append(time_block(engs[m], args.steps))
        for m in modes:
            eng = engs[m]
            prof = [eng.profile_step(0) for _ in range(3)][-1]
            kern = {}
            for n, t in prof:
                if n in KERNELS:
                    kern[n] = round(kern.get(n, 0.0) + t, 4)
            med = float(np.median(ms[m]))
            print(json.dumps({
                "mode": m, "ms_per_step": round(med, 4), "ms_per_step_blocks": [round(x, 4) for x in ms[m]],
                "spread_ms": round(float(np.max(ms[m]) - np.min(ms[m])), 4),
                "frames_per_s": round(B * T / (med * 1e-3), 1), "launches_per_step": eng.launches_per_step(),
                "kernels_ms": kern, "profiled_step_ms": round(sum(t for _, t in prof), 4),
                "config": {"batch": B, "trajectory": T, "num_action": A, "frames": "84x84x4", "cuda_graph": True,
                           "math_mode": 5, "batch_resident": True, "steps_per_block": args.steps,
                           "rounds": args.rounds,
                           "timing": "CUDA events on the compute stream around K back-to-back steps, modes alternating"},
                "gpu": info}))
    finally:
        for eng in engs.values():
            eng.close()


if __name__ == "__main__":
    main()
