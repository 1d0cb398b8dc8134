"""Actor-side latency of the Ape-X / A3C policy engine (`python tools/bench_apex_policy.py`), one H100, one JSON line.

For n in {1, 8, 16, 20, 40, 64} environments per call and both algos (84x84x4 frames, num_action 18):
  act_ms         median wall time of one synchronous NativeApexPolicy.act (epsilon = 0.1 drawn on the host) or
                 NativeA3CPolicy.act (uniforms drawn on the host) with graph replay, after warm-up of every n; the H2D
                 of the n frames and the rest of the inputs is counted inside the call, as is the host copy of the
                 outputs
  act_device_ms  median device time of the same calls (CUDA events around the input copy and the graph replay)
  learner_act_ms median wall time of drl_apex_act / drl_a3c_act on a NativeApexLearner / NativeA3CLearner(batch=n),
                 the learner-side path that apex.Agent / a3c.Agent.get_policy_and_action use (it synchronises the
                 learner's compute stream first and rebuilds the conv weight images after each learner step -- here
                 the learner takes no steps, so they are rebuilt only once); without the action rule
Then the Ape-X learner's B = 32 step with CUDA graphs (wall time per synchronous step, median) alone, and again while
a second thread drives NativeApexPolicy.act at n = 20 with one sync from the learner per trajectory = 20 calls.
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

A, B, TRAJ = 18, 32, 20


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # pragma: no cover - informational only
        return dict(gpu="unknown (%s)" % e)


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
    from distributed_reinforcement_learning_b200.a3c_learner import NativeA3CLearner
    from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET, NativeApexLearner
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy, NativeApexPolicy
    from distributed_reinforcement_learning_b200.model import actor_critic, apex_value
    from oracle import apex_torch as ax
    if _native.device_count() < 1:
        raise SystemExit("bench_apex_policy needs a CUDA device")
    np.random.seed(0)
    rng = np.random.default_rng(0)
    ns = (1, 8, 16, 20, 40, 64)
    data = {n: (rng.integers(0, 256, (n, 84, 84, 4), dtype=np.uint8), rng.integers(0, A, n).astype(np.int32))
            for n in ns}
    fams = dict(apex=(NativeApexPolicy, NativeApexLearner, apex_value.init_params(num_action=A),
                      lambda pol, n: pol.act(*data[n], epsilon=0.1)),
                a3c=(NativeA3CPolicy, NativeA3CLearner, actor_critic.init_params(num_action=A),
                     lambda pol, n: pol.act(*data[n])))
    res = {}
    for fam, (pcls, lcls, params, call) in fams.items():
        pol = pcls(64, num_action=A)
        pol.set_params(params)
        for n in ns:                                # warm-up of every n (eager pass + capture + replays)
            for _ in range(20):
                call(pol, n)
        res[fam] = {}
        for n in ns:
            dev = []

            def one():
                call(pol, n)
                dev.append(pol.last_act_ms())
            act_ms = median_ms(one, args.calls)
            lrn = lcls(batch=n, num_action=A)
            if fam == "apex":
                lrn.set_params(params, MAIN)
            else:
                lrn.set_params(params)
            for _ in range(20):
                lrn.act(*data[n])
            learner_ms = median_ms(lambda: lrn.act(*data[n]), args.calls)
            lrn.close()
            res[fam][str(n)] = dict(act_ms=round(act_ms, 4), act_device_ms=round(float(np.median(dev)), 4),
                                    learner_act_ms=round(learner_ms, 4), speedup=round(learner_ms / act_ms, 2))
        pol.close()
    # the Ape-X learner's step alone and under actor load
    params = apex_value.init_params(num_action=A)
    pol = NativeApexPolicy(64, num_action=A)
    pol.set_params(params)
    lrn = NativeApexLearner(batch=B, num_action=A, use_cuda_graph=True)
    lrn.set_params(params, MAIN)
    lrn.set_params(params, TARGET)
    t = ax.make_transitions(B, A=A, seed=1)
    targs = (t["state"], t["next_state"], t["previous_action"], t["action"], t["reward"], t["done"], t["is_weight"])
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
            if actor_calls[0] % TRAJ == 0:
                pol.sync_from(lrn)
            pol.act(*data[20], epsilon=0.1)
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
    out = dict(metric="Ape-X / A3C policy engine act latency (ms) vs drl_apex_act / drl_a3c_act; Ape-X learner step "
                      "under actor load",
               **gpu_info(), num_action=A, calls_per_n=args.calls, per_n=res,
               learner_step_ms=dict(shape="Ape-X B=%d cuda_graph" % B, alone=round(alone, 4),
                                    with_actor_n20=round(loaded, 4),
                                    slowdown_pct=round(100.0 * (loaded / alone - 1.0), 2),
                                    actor_calls_per_s=round(actor_calls[0] / wall, 1) if wall > 0 else None),
               note="act_ms counts the H2D of the n frames (28,224 B each) and the host copy of the outputs inside the "
                    "call; learner steps are synchronous (stage once, step + wait), median over %d steps" % args.steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
