"""Actor-side latency of the R2D2 policy engine (`python tools/bench_r2d2_policy.py`), one H100, one JSON line.

For n in {1, 8, 16, 40, 64} environments per call (84x84x1 frames, num_action 4, lstm_size 64):
  act_ms         median wall time of one synchronous NativeR2D2Policy.act (graph replay, epsilon = 0.1 drawn on the
                 host) after warm-up of every n; the H2D of the n frames and the rest of the inputs is counted inside
                 the call, as is the host copy of the outputs
  act_device_ms  median device time of the same calls (CUDA events around the input copy and the graph replay)
  learner_act_ms median wall time of drl_r2d2_act on a NativeR2D2Learner(batch=n, seq_len=2), the learner-side path
                 that r2d2.Agent.get_action uses (it synchronises the learner's compute stream first and rebuilds the
                 conv weight images after each learner step -- here the learner takes no steps, so they are rebuilt
                 only once)
Then the learner's B = 16, S = 80, burn-in 40 step with CUDA graphs (wall time per synchronous step, median) alone,
and again while a second thread drives act at n = 40 with one sync from the learner per seq_len = 80 calls.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

A, L, SEQ, BURN, B = 4, 64, 80, 40, 16


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # pragma: no cover - informational only
        return dict(gpu="unknown (%s)" % e)


def inputs(n, rng):
    return (rng.integers(0, 256, (n, 84, 84, 1), dtype=np.uint8), rng.integers(0, A, n).astype(np.int32),
            (rng.standard_normal((n, L)) * 0.5).astype(np.float32), rng.standard_normal((n, L)).astype(np.float32))


def median_ms(fn, calls):
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=500)
    ap.add_argument("--steps", type=int, default=60)
    args = ap.parse_args()
    from distributed_reinforcement_learning_b200 import _native
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET, NativeR2D2Learner
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
    from oracle import r2d2_torch as rt
    if _native.device_count() < 1:
        raise SystemExit("bench_r2d2_policy needs a CUDA device")
    np.random.seed(0)
    rng = np.random.default_rng(0)
    params = r2d2_lstm.init_params(num_action=A)
    pol = NativeR2D2Policy(64, num_action=A)
    pol.set_params(params)
    ns = (1, 8, 16, 40, 64)
    data = {n: inputs(n, rng) for n in ns}
    for n in ns:                                    # warm-up of every n (eager pass + capture + replays)
        for _ in range(20):
            pol.act(*data[n], epsilon=0.1)
    res = {}
    for n in ns:
        dev = []

        def one():
            pol.act(*data[n], epsilon=0.1)
            dev.append(pol.last_act_ms())
        act_ms = median_ms(one, args.calls)
        lrn = NativeR2D2Learner(batch=n, seq_len=2, burn_in=0, num_action=A)
        lrn.set_params(params, MAIN)
        for _ in range(20):
            lrn.act(*data[n])
        learner_ms = median_ms(lambda: lrn.act(*data[n]), args.calls)
        lrn.close()
        res[str(n)] = dict(act_ms=round(act_ms, 4), act_device_ms=round(float(np.median(dev)), 4),
                           learner_act_ms=round(learner_ms, 4), speedup=round(learner_ms / act_ms, 2))
    # the learner's step alone and under actor load
    lrn = NativeR2D2Learner(batch=B, seq_len=SEQ, burn_in=BURN, num_action=A, use_cuda_graph=True)
    lrn.set_params(params, MAIN)
    lrn.set_params(params, TARGET)
    b = rt.make_sequences(B, S=SEQ, A=A, seed=1)
    targs = (b["state"], b["previous_action"], b["action"], b["h"][:, 0], b["c"][:, 0], b["reward"], b["done"],
             b["weight"])
    lrn.stage(0, *targs)
    lrn.stage(1, *targs)

    def learner_steps(k):
        ts = []
        for s in range(k):
            t0 = time.perf_counter()
            lrn.step(s % 2)
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts)) * 1e3
    learner_steps(10)
    alone = learner_steps(args.steps)
    stop, actor_calls = threading.Event(), [0]

    def actor():
        while not stop.is_set():
            if actor_calls[0] % SEQ == 0:
                pol.sync_from(lrn)
            pol.act(*data[40], epsilon=0.1)
            actor_calls[0] += 1
    th = threading.Thread(target=actor)
    th.start()
    time.sleep(0.2)
    t0 = time.perf_counter()
    loaded = learner_steps(args.steps)
    wall = time.perf_counter() - t0
    stop.set()
    th.join()
    lrn.close()
    pol.close()
    out = dict(metric="R2D2 policy engine act latency (ms) vs drl_r2d2_act; learner step under actor load",
               **gpu_info(), calls_per_n=args.calls, per_n=res,
               learner_step_ms=dict(shape="B=%d S=%d burn_in=%d cuda_graph" % (B, SEQ, BURN), alone=round(alone, 4),
                                    with_actor_n40=round(loaded, 4),
                                    slowdown_pct=round(100.0 * (loaded / alone - 1.0), 2),
                                    actor_calls_per_s=round(actor_calls[0] / wall, 1) if wall > 0 else None),
               note="act_ms counts the H2D of the n frames (7,056 B each) and the host copy of the outputs inside the "
                    "call; learner steps are synchronous (stage once, step + wait), median over %d steps" % args.steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
