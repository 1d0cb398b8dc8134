"""R2D2 learner step with the reference's targets and priorities (one-step double-Q, |mean td|) against the R2D2 paper's
(n = 5 step targets, priority 0.9 max |td| + 0.1 mean |td|, DESIGN.md section 22).  B = 16 sequences of S = 80 steps,
burn-in 40, 84x84x1 frames, A = 4, math mode 2, CUDA graphs, a device-resident batch (both staged slots filled once,
then stepped alternately), at lstm_size 64 and 512.

The two modes are timed in alternating blocks of K back-to-back steps (CUDA events on each learner's compute stream), so
the spread between blocks shows beside the difference between modes.  Then one profiled step per mode gives the TD
kernel's time (r2d2_td_kernel by default, r2d2_td_nstep_kernel otherwise).  Prints the card's name, power limit and
maximum SM clock (read in the same run), then one JSON line per width and mode.

    python tools/bench_r2d2_nstep.py [--steps 20] [--warmup 5] [--rounds 7] [--lstm-sizes 64,512]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_impala_recurrent import gpu_info  # noqa: E402

B, S, BI, A = 16, 80, 40, 4
MODES = {"reference": dict(n_step=1, priority_eta=None), "nstep5_eta0.9": dict(n_step=5, priority_eta=0.9)}


def make_learner(L, batch, main, target, **kw):
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    eng = NativeR2D2Learner(batch=B, seq_len=S, burn_in=BI, num_action=A, lstm_size=L, use_cuda_graph=True,
                            math_mode=2, **kw)
    eng.set_params(main, MAIN)
    eng.set_params(target, TARGET)
    for slot in range(2):
        eng.stage(slot, batch["state"], batch["previous_action"], batch["action"], batch["h"][:, 0], batch["c"][:, 0],
                  batch["reward"], batch["done"], batch["weight"])
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
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--lstm-sizes", default="64,512")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_r2d2_nstep needs a CUDA device")
    torch.cuda.set_device(0)
    from oracle import r2d2_torch as rt
    info = gpu_info()
    print(json.dumps({"gpu": info}))
    for L in (int(x) for x in args.lstm_sizes.split(",")):
        kw = dict(num_action=A, lstm_size=L)
        batch = rt.make_sequences(B, S=S, A=A, L=L, seed=2468)
        main_p = rt.flatten_params(rt.init_params(0, torch.float32, **kw))
        target_p = rt.flatten_params(rt.init_params(1, torch.float32, **kw))
        engs = {m: make_learner(L, batch, main_p, target_p, **c) for m, c in MODES.items()}
        try:
            for m in MODES:
                for i in range(max(args.warmup, 3)):
                    engs[m].step(i % 2)
            ms = {m: [] for m in MODES}
            for _ in range(args.rounds):
                for m in MODES:
                    ms[m].append(time_block(engs[m], args.steps))
            for m in MODES:
                eng = engs[m]
                prof = [eng.profile_step(0) for _ in range(3)][-1]
                td_ms = sum(t for n, t in prof if n == "td_target_loss")
                med = float(np.median(ms[m]))
                print(json.dumps({
                    "lstm_size": L, "mode": m, **MODES[m], "ms_per_step": round(med, 4),
                    "ms_per_step_blocks": [round(x, 4) for x in ms[m]],
                    "spread_ms": round(float(np.max(ms[m]) - np.min(ms[m])), 4),
                    "launches_per_step": eng.launches_per_step(), "td_kernel_ms": round(td_ms, 4),
                    "profiled_step_ms": round(sum(t for _, t in prof), 4),
                    "config": {"batch": B, "seq_len": S, "burn_in": BI, "num_action": A, "frames": "84x84x1",
                               "cuda_graph": True, "math_mode": 2, "batch_resident": True,
                               "steps_per_block": args.steps, "rounds": args.rounds,
                               "timing": "CUDA events on the compute stream around K back-to-back steps, modes "
                                         "alternating"},
                    "gpu": info}))
        finally:
            for eng in engs.values():
                eng.close()


if __name__ == "__main__":
    main()
