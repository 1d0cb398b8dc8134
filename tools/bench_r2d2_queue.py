"""The co-located R2D2 actor -> replay -> learner loop with the sequence queue on the host and on the GPU
(`python tools/bench_r2d2_queue.py`), one H100, one JSON line per actor count.

Both arms run the loop of train_r2d2.py in one process, alternating blocks of iterations:
  host    R2D2VectorActor + buffer_queue.R2D2FIFOQueue (R2D2TrajectoryBuffer, append_to_queue) +
          DeviceMemory.add of sample_batch (np.stack + one H2D of the batch) + Agent.train_from_memory
  device  R2D2VectorActor + buffer_queue.R2D2DeviceFIFOQueue (the policy's recorder; one commit of reward and done per
          unroll) + DeviceMemory.add_from_queue (the learner and the store read the queue slot) + train_from_memory
One iteration = one unroll of n environments (the learner's parameters synced into the policy first, S batched acts),
the ingest of every full batch the queue then holds (n = 16: one; n = 40: 2.5 on average), and one training step once
more than two batches have been ingested (train_r2d2.py:97-165).  The environments are cheap seeded synthetic ones
(frames drawn from a fixed pool), so the loop measures the engine, the queue, the memory and the learner, not an
emulator.  S = 15, burn-in 7, 84x84x1 frames, A = 4, B = 16, queue_size 128, lstm 64, CUDA graphs on; both memories are
pre-filled with the same 512 sequences.  Reported per arm: ms per iteration (median, p10-p90) split into actor, ingest
and train time, environment frames per second, H2D bytes per iteration computed from shapes, and kernels and copies
per iteration from a separate torch.profiler run.  The first K iterations of both arms start from the same seeds and
parameters; their losses, |td|, sampled indices and final parameters must be bit-equal (bit_equal).
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

S, BURN_IN, A, L, B, QUEUE, CAPACITY, PREFILL = 15, 7, 4, 64, 16, 128, 2048, 512
SHAPE = (84, 84, 1)
FRAME = 84 * 84 * 1
SEQ_H2D = S * (FRAME + 4 + 4 + 4 + 1) + 2 * 4 * L   # one sequence as DeviceMemory.add uploads it: 106,547 B
ACT_H2D = FRAME + 4 + 4 * L + 4 * L + 4               # one act row: frame, previous action, h, c, explore: 7,576 B


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


def make_agent(name, params, target):
    from distributed_reinforcement_learning_b200.agent import r2d2
    ag = r2d2.Agent(S, BURN_IN, list(SHAPE), A, L, 0.997, 1e-4, 1e-4, 1e9, 40.0, name, name)
    ag.use_cuda_graph = True
    ag._main, ag._target = params.copy(), target.copy()
    z = np.zeros_like(params)
    ag._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    ag._get_engine(B)
    return ag


def prefill(memory, seed):
    rng = np.random.default_rng(seed)
    for _ in range(PREFILL // B):
        memory.add(rng.integers(0, 256, (B, S) + SHAPE, dtype=np.uint8), rng.integers(0, A, (B, S)),
                   rng.integers(0, A, (B, S)), np.zeros((B, L), np.float32), np.zeros((B, L), np.float32),
                   rng.integers(0, 2, (B, S)).astype(np.float32), rng.random((B, S)) < 0.01)


class Arm:
    def __init__(self, kind, n, params, target, seed):
        from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
        from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue as bq
        from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
        self.kind, self.n = kind, n
        self.agent = make_agent("bench_r2q_%s_%d" % (kind, n), params, target)
        self.memory = self.agent.device_memory(CAPACITY)
        prefill(self.memory, seed)
        cls = bq.R2D2FIFOQueue if kind == "host" else bq.R2D2DeviceFIFOQueue
        self.queue = cls(S, SHAPE, A, QUEUE, B, n, L)
        self.policy = NativeR2D2Policy(64, num_action=A, lstm_size=L, input_shape=SHAPE, use_cuda_graph=True)
        self.actor = R2D2VectorActor(self.policy, [PoolEnv(seed * 1000 + i) for i in range(n)], self.queue, S,
                                     learner=self.agent)
        self.buffer_step = 0
        self.out = []

    def ingest(self):
        if self.kind == "host":
            b = self.queue.sample_batch()
            self.memory.add(b.state, b.previous_action, b.action, b.previous_h, b.previous_c, b.reward, b.done)
        else:
            self.memory.add_from_queue(self.queue)
        self.buffer_step += B

    def iteration(self):
        t0 = time.perf_counter()
        self.actor.run_unroll()
        t1 = time.perf_counter()
        ingests = 0
        while self.queue.get_size() >= B:
            self.ingest()
            ingests += 1
        t2 = time.perf_counter()
        trains = 0
        if self.buffer_step > 2 * B:
            loss, td = self.agent.train_from_memory(self.memory, B)
            self.out.append((loss, np.array(td), self.memory.last_sample()[0].copy()))
            trains = 1
        return t1 - t0, t2 - t1, time.perf_counter() - t2, ingests, trains


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


def run(n, blocks, iters, parity, profile_iters, seed):
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    from distributed_reinforcement_learning_b200.r2d2_learner import MAIN, TARGET
    kw = dict(num_action=A, lstm_size=L, input_shape=SHAPE)
    params, target = r2d2_lstm.init_params(seed, **kw), r2d2_lstm.init_params(seed + 1, **kw)
    arms = {}
    for kind in ("host", "device"):
        np.random.seed(seed)
        random.seed(seed)
        arms[kind] = Arm(kind, n, params, target, seed)
        for _ in range(parity):
            arms[kind].iteration()
    h, d = arms["host"], arms["device"]
    bit_equal = len(h.out) == len(d.out) > 0 and all(
        lh == ld and np.array_equal(th, td) and np.array_equal(ih, idd)
        for (lh, th, ih), (ld, td, idd) in zip(h.out, d.out)) and \
        all(np.array_equal(h.agent._engine.get_params(w), d.agent._engine.get_params(w)) for w in (MAIN, TARGET))
    n_parity_steps = len(h.out)
    res = {k: dict(actor=[], ingest=[], train=[], total=[], ingests=0, trains=0, iters=0) for k in arms}
    for _ in range(blocks):
        for kind, arm in arms.items():
            r = res[kind]
            for _ in range(iters):
                ta, ti, tt, ni, nt = arm.iteration()
                r["actor"].append(ta)
                r["ingest"].append(ti)
                r["train"].append(tt)
                r["total"].append(ta + ti + tt)
                r["ingests"] += ni
                r["trains"] += nt
                r["iters"] += 1
    out = {}
    for kind, r in res.items():
        ingests_per_iter = r["ingests"] / r["iters"]
        trains_per_iter = r["trains"] / r["iters"]
        ingest_h2d = B * SEQ_H2D if kind == "host" else 0
        commit_h2d = 0 if kind == "host" else n * S * 5 + 4
        out[kind] = dict(
            ms_per_iter=pct(r["total"], 50), ms_p10=pct(r["total"], 10), ms_p90=pct(r["total"], 90),
            actor_ms=pct(r["actor"], 50), ingest_ms=pct(r["ingest"], 50), train_ms=pct(r["train"], 50),
            ingests_per_iter=ingests_per_iter, trains_per_iter=trains_per_iter,
            env_frames_per_s=n * S * r["iters"] / float(np.sum(r["total"])),
            h2d_bytes_per_iter=int(n * S * ACT_H2D + commit_h2d + ingests_per_iter * ingest_h2d
                                   + trains_per_iter * B * 8))
    for kind, arm in arms.items():
        try:
            out[kind].update(profile(arm, profile_iters))
        except Exception as e:   # pragma: no cover - the profiler is optional
            out[kind]["profile_error"] = str(e)
    speedup = out["host"]["ms_per_iter"] / out["device"]["ms_per_iter"]
    return dict(bench="r2d2_queue", n=n, seq_len=S, burn_in=BURN_IN, num_action=A, batch=B, queue_size=QUEUE,
                capacity=CAPACITY, prefill=PREFILL, cuda_graph=True, blocks=blocks, iters_per_block=iters,
                parity_iters=parity, parity_train_steps=n_parity_steps, bit_equal=bool(bit_equal),
                host=out["host"], device=out["device"], speedup_per_iter=speedup, **gpu_info())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="16,40", help="environments per actor (comma-separated)")
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--iters", type=int, default=20, help="iterations per arm per block")
    ap.add_argument("--parity", type=int, default=12, help="K: iterations compared from the same seeds")
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
