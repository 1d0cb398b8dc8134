"""The co-located IMPALA actor -> learner loop with the trajectory queue on the host and on the GPU
(`python tools/bench_impala_queue.py`), one H100, one JSON line per actor count.

Both arms run the loop of train_impala.py in one process, alternating blocks of iterations:
  host    VectorActor + buffer_queue.FIFOQueue (UnrolledTrajectory, append_to_queue into the pinned ring) +
          Agent.train on sample_batch (H2D of the whole batch)
  device  VectorActor + buffer_queue.DeviceFIFOQueue (the policy's recorder; one commit of reward and done per unroll) +
          Agent.train_from_queue (device-to-device staging)
One iteration = one unroll of n environments (the learner's parameters synced into the policy first, T batched acts)
plus every learner step the queue then holds a batch for (n = 32: one; n = 20: one every 1.6 iterations).  The
environments are cheap seeded synthetic ones (frames drawn from a fixed pool), so the loop measures the engine, the
queue and the learner, not an emulator.  T = 20, A = 18, B = 32, lstm 256, 84x84x4 frames, CUDA graphs on.
Reported per arm: ms per iteration (median, p10-p90) split into actor and learner time, environment frames per second,
H2D bytes per iteration computed from shapes, kernels and copies per iteration from a separate torch.profiler run,
and the learner step time alone and while the other arm's actors record.  The first K iterations of both arms start
from the same seeds and parameters; their losses and final parameters must be bit-equal (bit_equal).
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

T, A, L, B, QUEUE = 20, 18, 256, 32, 128
SHAPE = (84, 84, 4)
FRAME = 84 * 84 * 4
ROW_BYTES = FRAME + 4 + 1 + 4 * A + 4 + 4 + 4 * L + 4 * L     # one trajectory step-row, 30,357 B at A = 18
ACT_H2D = FRAME + 4 + 4 * L + 4 * L + 8                        # one act row: frame, previous action, h, c, uniform


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # pragma: no cover - informational only
        return dict(gpu="unknown (%s)" % e)


class PoolEnv:
    """A seeded synthetic environment: frames from a shared pool of 64, rewards in {0, 1}, a life lost now and then,
    episodes of a few hundred steps."""
    POOL = None

    def __init__(self, seed):
        if PoolEnv.POOL is None:
            PoolEnv.POOL = np.random.default_rng(0).integers(0, 256, (64,) + SHAPE, dtype=np.uint8)
        self.rng = np.random.RandomState(seed)

    def reset(self):
        self.lives, self.t = 5, 0
        return PoolEnv.POOL[self.rng.randint(64)]

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.01:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 400
        return PoolEnv.POOL[self.rng.randint(64)], float(self.rng.rand() < 0.1), done, {"ale.lives": self.lives}


def make_agent(name, params):
    from distributed_reinforcement_learning_b200.agent import impala
    ag = impala.Agent(trajectory=T, input_shape=SHAPE, num_action=A, lstm_hidden_size=L, discount_factor=0.99,
                      start_learning_rate=0.0006, end_learning_rate=0.0, learning_frame=1e9, baseline_loss_coef=1.0,
                      entropy_coef=0.05, gradient_clip_norm=40.0, reward_clipping="abs_one", model_name=name,
                      learner_name=name)
    ag.use_cuda_graph = True
    ag._ensure_init()
    ag._params = params.copy()
    ag._get_engine(B)
    return ag


class Arm:
    def __init__(self, kind, n, params, seed):
        from distributed_reinforcement_learning_b200.actor import VectorActor
        from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue as bq
        from distributed_reinforcement_learning_b200.policy import NativePolicy
        self.kind, self.n = kind, n
        self.agent = make_agent("bench_%s_%d" % (kind, n), params)
        cls = bq.FIFOQueue if kind == "host" else bq.DeviceFIFOQueue
        self.queue = cls(T, SHAPE, A, QUEUE, B, n, L)
        self.policy = NativePolicy(64, num_action=A, use_cuda_graph=True)
        self.actor = VectorActor(self.policy, [PoolEnv(seed * 1000 + i) for i in range(n)], self.queue, T, [A] * n,
                                 learner=self.agent)
        self.losses = []

    def train(self):
        if self.kind == "host":
            b = self.queue.sample_batch()
            return self.agent.train(b.state, b.reward, b.action, b.done, b.behavior_policy, b.previous_action,
                                    b.previous_h, b.previous_c)
        return self.agent.train_from_queue(self.queue)

    def iteration(self):
        t0 = time.perf_counter()
        self.actor.run_unroll()
        t1 = time.perf_counter()
        steps = 0
        while self.queue.get_size() >= B:
            self.losses.append(self.train())
            steps += 1
        return t1 - t0, time.perf_counter() - t1, steps


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def profile(arm, iters):
    """Kernels / copies per iteration from torch.profiler (its own run)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            arm.iteration()
        torch.cuda.synchronize()
    kernels, copies, h2d = 0, 0, 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
            copies += 1
            h2d += "HtoD" in e.name
        else:
            kernels += 1
    return dict(kernels_per_iter=kernels / iters, copies_per_iter=copies / iters, h2d_copies_per_iter=h2d / iters)


def learner_step_ms(dev_arm, other, steps):
    """ms per train_from_queue step from a pre-filled device queue: alone, then while `other`'s actor records."""
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.policy import NativePolicy
    q = DeviceFIFOQueue(T, SHAPE, A, steps * B, B, 32, L)
    pol = NativePolicy(64, num_action=A)
    dev_arm.agent.sync_policy(pol)
    rec = pol.recorder(q, 32)
    rng = np.random.RandomState(5)
    zeros = np.zeros((32, L), np.float32)

    def fill():
        for _ in range(steps):
            for _ in range(T):
                rec.act(PoolEnv.POOL[rng.randint(64, size=32)], rng.randint(0, A, 32), zeros, zeros)
            rec.commit(np.zeros((32, T), np.float32), np.zeros((32, T), np.bool_))

    def timed():
        ts = []
        for _ in range(steps):
            t0 = time.perf_counter()
            dev_arm.agent.train_from_queue(q)
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts) * 1e3)

    fill()
    alone = timed()
    fill()
    stop = threading.Event()

    def actor_loop():
        # the host arm's actor keeps acting and pushing into its ring, drained without training so it never blocks
        while not stop.is_set():
            other.actor.run_unroll()
            while other.queue.get_size() >= B:
                other.queue.sample_batch()

    th = threading.Thread(target=actor_loop)
    th.start()
    time.sleep(0.2)
    busy = timed()
    stop.set()
    th.join()
    rec.close()
    pol.close()
    q.close()
    return alone, busy


def run(n, blocks, iters, parity, profile_iters, seed):
    from distributed_reinforcement_learning_b200.model import impala_actor_critic
    params = impala_actor_critic.init_params(seed=seed, num_action=A, lstm_hidden_size=L, input_shape=SHAPE)
    arms = {}
    for kind in ("host", "device"):
        np.random.seed(seed)
        arms[kind] = Arm(kind, n, params, seed)
        for _ in range(parity):
            arms[kind].iteration()
    h, d = arms["host"], arms["device"]
    bit_equal = h.losses == d.losses and len(h.losses) > 0 and \
        np.array_equal(h.agent._engine.get_params(), d.agent._engine.get_params())
    n_parity_steps = len(h.losses)
    res = {k: dict(actor=[], learner=[], total=[], steps=0, iters=0) for k in arms}
    for _ in range(blocks):
        for kind, arm in arms.items():
            r = res[kind]
            for _ in range(iters):
                ta, tl, st = arm.iteration()
                r["actor"].append(ta)
                r["learner"].append(tl)
                r["total"].append(ta + tl)
                r["steps"] += st
                r["iters"] += 1
    out = {}
    for kind, r in res.items():
        steps_per_iter = r["steps"] / r["iters"]
        batch_h2d = B * T * ROW_BYTES if kind == "host" else 0
        rd_h2d = 0 if kind == "host" else n * T * 5 + 4 * T
        out[kind] = dict(
            ms_per_iter=pct(r["total"], 50), ms_p10=pct(r["total"], 10), ms_p90=pct(r["total"], 90),
            actor_ms=pct(r["actor"], 50), learner_ms_per_iter=float(np.mean(r["learner"]) * 1e3),
            learner_steps_per_iter=steps_per_iter,
            env_frames_per_s=n * T * r["iters"] / float(np.sum(r["total"])),
            h2d_bytes_per_iter=int(n * T * ACT_H2D + rd_h2d + steps_per_iter * batch_h2d))
    for kind, arm in arms.items():
        try:
            out[kind].update(profile(arm, profile_iters))
        except Exception as e:   # pragma: no cover - the profiler is optional
            out[kind]["profile_error"] = str(e)
    alone, busy = learner_step_ms(d, h, 10)
    out["device"].update(learner_step_ms_alone=alone, learner_step_ms_with_host_actor=busy)
    speedup = out["host"]["ms_per_iter"] / out["device"]["ms_per_iter"]
    return dict(bench="impala_queue", n=n, trajectory=T, num_action=A, batch=B, queue_size=QUEUE, cuda_graph=True,
                blocks=blocks, iters_per_block=iters, parity_iters=parity, parity_learner_steps=n_parity_steps,
                bit_equal=bool(bit_equal), host=out["host"], device=out["device"],
                speedup_per_iter=speedup, **gpu_info())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="32,20", help="environments per actor (comma-separated)")
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--iters", type=int, default=20, help="iterations per arm per block")
    ap.add_argument("--parity", type=int, default=20, help="K: iterations compared from the same seeds")
    ap.add_argument("--profile-iters", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    from distributed_reinforcement_learning_b200 import _native as N
    if N.device_count() < 1:
        raise SystemExit("needs a CUDA device (no CPU fallback)")
    ok = True
    for n in [int(x) for x in a.n.split(",")]:
        r = run(n, a.blocks, a.iters, a.parity, a.profile_iters, a.seed)
        ok = ok and r["bit_equal"]
        print(json.dumps(r), flush=True)
    if not ok:
        raise SystemExit("bit check failed: the host and device arms diverged")


if __name__ == "__main__":
    main()
