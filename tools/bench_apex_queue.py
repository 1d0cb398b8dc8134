"""The co-located Ape-X actor -> replay -> learner loop with the transition queue on the host and on the GPU
(`python tools/bench_apex_queue.py`), one H100, one JSON line per actor count.

Both arms run the loop of train_apex.py in one process, alternating blocks of iterations:
  host    ApexVectorActor + n LocalBuffer(1e4) + buffer_queue.ApexFIFOQueue (append_to_queue of every sample) +
          DeviceMemory.add of sample_batch(1) (np.stack + one H2D of the record) + Agent.train_from_memory
  device  ApexVectorActor + DeviceLocalBuffers(n, 1e4) + buffer_queue.ApexDeviceFIFOQueue (one append per step, one
          push per sample, on the device) + DeviceMemory.add_from_queue (the learner and the store read the queue slot)
          + train_from_memory
One iteration = one unroll of n environments (the learner's parameters synced into the policy first, T batched acts);
once the buffers hold more than 3T transitions every environment step pushes one record of T transitions.  Then, as in
the learner loop of train_apex.py:94-155, every queued record is ingested, each ingest followed by one training step
once more than 10 records have been ingested.  The queue holds n * T records, one unroll's worth, so that this
single-threaded loop never blocks on a full queue (the reference's queue_size 32 throttles actor processes instead).
The environments are cheap seeded synthetic ones (frames drawn from a fixed pool, an episode end every few hundred
steps), so the loop measures the engine, the buffers, the queue, the memory and the learner, not an emulator.
T = 32, A = 4, B = 32, 84x84x4 frames, buffer capacity 1e4, memory capacity 2^16, CUDA graphs on (the reference's
configuration otherwise).  Reported per arm: environment steps per second, ms per iteration (median, p10-p90) split
into actor, ingest and train time, ingest ms per record, train ms per step, and the H2D bytes computed from shapes.
The first K iterations of both arms start from the same seeds and parameters; their losses, |td|, sampled indices and
final parameters must be bit-equal (bit_equal).
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

T, A, B, BUFFER, CAPACITY = 32, 4, 32, 10000, 1 << 16
SHAPE = (84, 84, 4)
FRAME = 84 * 84 * 4
# one record as DeviceMemory.add uploads it: 2T frames, previous_action + action, reward, done and the unit weights
RECORD_H2D = 2 * T * FRAME + 2 * T * 4 + T * 4 + T + T * 4   # 1,806,880 B


def append_h2d(n, uploaded_states):
    """One DeviceLocalBuffers.append: the scalar block (five 256-aligned [n] fields), n next_state frames and the
    states the device does not hold."""
    return 5 * (-(-n * 4 // 256) * 256) + (n + uploaded_states) * FRAME


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
        self.resets = 0

    def reset(self):
        self.lives, self.t = 5, 0
        self.resets += 1
        return PoolEnv.POOL[self.rng.randint(64)]

    def step(self, a):
        self.t += 1
        if self.rng.rand() < 0.01:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 400
        return PoolEnv.POOL[self.rng.randint(64)], float(self.rng.rand() < 0.1), done, {"ale.lives": self.lives}


def make_agent(name, params, target):
    from distributed_reinforcement_learning_b200.agent import apex
    ag = apex.Agent(list(SHAPE), A, 0.99, 40.0, "abs_one", 1e-4, 0.0, 1e14, name, name)
    ag.use_cuda_graph = True
    ag._main, ag._target = params.copy(), target.copy()
    z = np.zeros_like(params)
    ag._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    ag._get_engine(B)
    return ag


class Arm:
    def __init__(self, kind, n, params, target, seed):
        from distributed_reinforcement_learning_b200.actor import ApexVectorActor
        from distributed_reinforcement_learning_b200.apex_policy import NativeApexPolicy
        from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue as bq
        self.kind, self.n = kind, n
        self.agent = make_agent("bench_aq_%s_%d" % (kind, n), params, target)
        self.memory = self.agent.device_memory(CAPACITY)
        cls = bq.ApexFIFOQueue if kind == "host" else bq.ApexDeviceFIFOQueue
        self.queue = cls(T, SHAPE, A, n * T, B, n)
        self.policy = NativeApexPolicy(64, num_action=A, input_shape=SHAPE, use_cuda_graph=True)
        self.envs = [PoolEnv(seed * 1000 + i) for i in range(n)]
        self.actor = ApexVectorActor(self.policy, self.envs, self.queue, T, [A] * n, learner=self.agent,
                                     buffer_capacity=BUFFER)
        self.buffer_step = 0
        self.out = []

    def ingest(self):
        if self.kind == "host":
            b = self.queue.sample_batch(1)
            self.memory.add(b.state[0], b.next_state[0], b.previous_action[0], b.action[0], b.reward[0], b.done[0])
        else:
            self.memory.add_from_queue(self.queue)
        self.buffer_step += 1

    def iteration(self):
        """-> actor s, ingest s, train s, records, train steps, states uploaded by the device appends."""
        resets0 = sum(e.resets for e in self.envs)
        t0 = time.perf_counter()
        self.actor.run_unroll()
        ta = time.perf_counter() - t0
        ti = tt = 0.0
        records = trains = 0
        while self.queue.get_size():
            t1 = time.perf_counter()
            self.ingest()
            self.memory.total()      # waits for the ingest's device work (the same 8-byte read in both arms)
            t2 = time.perf_counter()
            ti += t2 - t1
            records += 1
            if self.buffer_step > 10:
                loss, td = self.agent.train_from_memory(self.memory, B)
                self.out.append((loss, np.array(td), self.memory.last_sample()[0].copy()))
                tt += time.perf_counter() - t2
                trains += 1
        return ta, ti, tt, records, trains, sum(e.resets for e in self.envs) - resets0


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def run(n, blocks, iters, parity, seed):
    from distributed_reinforcement_learning_b200.apex_learner import MAIN, TARGET
    from distributed_reinforcement_learning_b200.model import apex_value
    kw = dict(num_action=A, input_shape=SHAPE)
    params, target = apex_value.init_params(seed, **kw), apex_value.init_params(seed + 1, **kw)
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
    res = {k: dict(actor=[], ingest=0.0, train=0.0, total=[], records=0, trains=0, iters=0, uploads=0) for k in arms}
    for _ in range(blocks):
        for kind, arm in arms.items():
            r = res[kind]
            for _ in range(iters):
                ta, ti, tt, nr, nt, resets = arm.iteration()
                r["actor"].append(ta)
                r["total"].append(ta + ti + tt)
                r["ingest"] += ti
                r["train"] += tt
                r["records"] += nr
                r["trains"] += nt
                r["iters"] += 1
                r["uploads"] += resets
    out = {}
    for kind, r in res.items():
        steps = n * T * r["iters"]
        if kind == "host":
            h2d_per_iter = r["records"] / r["iters"] * RECORD_H2D
        else:   # T appends per unroll; a state crosses PCIe only after an episode reset
            h2d_per_iter = T * append_h2d(n, 0) + r["uploads"] / r["iters"] * FRAME
        out[kind] = dict(
            env_steps_per_s=steps / float(np.sum(r["total"])),
            ms_per_iter=pct(r["total"], 50), ms_p10=pct(r["total"], 10), ms_p90=pct(r["total"], 90),
            actor_ms=pct(r["actor"], 50),
            ingest_ms_per_record=1e3 * r["ingest"] / max(r["records"], 1),
            train_ms_per_step=1e3 * r["train"] / max(r["trains"], 1),
            records_per_iter=r["records"] / r["iters"], trains_per_iter=r["trains"] / r["iters"],
            record_h2d_bytes=RECORD_H2D if kind == "host" else 0,
            queue_h2d_bytes_per_iter=int(h2d_per_iter))
    speedup = out["device"]["env_steps_per_s"] / out["host"]["env_steps_per_s"]
    return dict(bench="apex_queue", n=n, trajectory=T, num_action=A, batch=B, buffer_capacity=BUFFER,
                queue_size=n * T, memory_capacity=CAPACITY, cuda_graph=True, blocks=blocks, iters_per_block=iters,
                parity_iters=parity, parity_train_steps=n_parity_steps, bit_equal=bool(bit_equal),
                host=out["host"], device=out["device"], env_steps_speedup=speedup, **gpu_info())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="1,16,20", help="environments per actor (comma-separated)")
    ap.add_argument("--blocks", type=int, default=2)
    ap.add_argument("--iters", type=int, default=2, help="iterations per arm per block")
    ap.add_argument("--parity", type=int, default=5, help="K: iterations compared from the same seeds (>= 4: the "
                                                            "first 3 unrolls fill the buffers without pushing)")
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    from distributed_reinforcement_learning_b200 import _native as N
    if N.device_count() < 1:
        raise SystemExit("needs a CUDA device (no CPU fallback)")
    ok = True
    for n in [int(x) for x in a.n.split(",")]:
        r = run(n, a.blocks, a.iters, a.parity, a.seed)
        ok = ok and r["bit_equal"]
        print(json.dumps(r), flush=True)
    if not ok:
        raise SystemExit("bit check failed: the host and device arms diverged")


if __name__ == "__main__":
    main()
