"""The R2D2 learner loop with the replay memory on the host and on the GPU (`python tools/bench_r2d2_replay.py`), one
H100, one JSON line.

Both arms run the learner branch of train_r2d2.py:87-165 at the reference configuration (batch 16, seq_len 15,
burn_in 7, 84x84x1 frames, lstm 64, num_action 4, capacity 1e5 pre-filled) in the same process, alternating blocks of
iterations:
  host    r2d2.Agent + buffer_queue.Memory, the loop as the reference writes it: 16 get_td_error calls of one sequence
          each, 16 Memory.add, then Memory.sample, seven Python lists, train (np.stack + H2D + step), 16 Memory.update
  device  r2d2.Agent.device_memory + DeviceMemory.add (ingest of the whole queued batch) + Agent.train_from_memory
One iteration = one queued batch of 16 sequences ingested + one training step.  The memory is filled, and the batches
drawn, from a pool of 256 distinct synthetic sequences (the host arm stores views of the pool's arrays).
Reported per arm: wall ms per iteration (median), its ingest / train split, sequences trained per second (16 per
iteration), and from a separate torch.profiler run of a few iterations the kernels and copies per iteration and the
device time of the replay kernels (sample, sequence gather, tree update, sequence store).  The device arm's ingest only
enqueues work; its device time lands in the train call that follows, so only the sum is comparable.  Also: for the
first K iterations from the same seeds and the same parameters, with the host arm's priorities taken from the
learner's batched |td| as the device ingest computes them, whether both arms sampled the same indices, and the largest
relative difference of their losses.
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

A, B, S, BURN_IN, L, POOL = 4, 16, 15, 7, 64, 256
SHAPE = (84, 84, 1)
TARGET_EVERY = 2500          # train_r2d2.py:164


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # pragma: no cover - informational only
        return dict(gpu="unknown (%s)" % e)


def make_pool(seed):
    rng = np.random.default_rng(seed)
    return dict(state=rng.integers(0, 256, (POOL, S) + SHAPE, dtype=np.uint8),
                previous_action=rng.integers(0, A, (POOL, S)).astype(np.int32),
                action=rng.integers(0, A, (POOL, S)).astype(np.int32),
                reward=(rng.standard_normal((POOL, S)) * 2).astype(np.float32), done=rng.random((POOL, S)) < 0.05,
                previous_h=(rng.standard_normal((POOL, S, L)) * 0.3).astype(np.float32),
                previous_c=(rng.standard_normal((POOL, S, L)) * 0.3).astype(np.float32))


FIELDS = ("state", "previous_action", "action", "reward", "done", "previous_h", "previous_c")   # Memory record order


def queued(pool, k):
    """One R2D2FIFOQueue.sample_batch() of B sequences, as a dict of [B, ...] arrays."""
    lo = (k * B) % POOL
    return {f: pool[f][lo:lo + B] for f in FIELDS}


def make_agent(name, params, graph):
    from distributed_reinforcement_learning_b200.agent import r2d2
    a = r2d2.Agent(S, BURN_IN, list(SHAPE), A, L, 0.997, 1e-4, 0.0, 1e9, 40.0, name, name)
    a.use_cuda_graph = graph
    a._main, a._target = params[0].copy(), params[1].copy()
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    a.main_to_target()
    return a


class HostArm:
    """train_r2d2.py:87-165 as written, on r2d2.Agent + buffer_queue.Memory.  batched_priorities: the priorities are the
    learner's batched |td| of each queued batch (the device ingest's arithmetic) instead of 16 get_td_error calls."""

    def __init__(self, agent, capacity, pool, errors):
        from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
        self.agent, self.memory, self.train_step = agent, Memory(capacity), 0
        self.batched_priorities = False
        for i, e in enumerate(errors):
            j = i % POOL
            self.memory.add(e, [pool[f][j] for f in FIELDS])
        agent._get_engine(B)

    def ingest(self, q):
        if self.batched_priorities:
            td = self.agent._engine.td_error(q["state"], q["previous_action"], q["action"], q["previous_h"][:, 0],
                                             q["previous_c"][:, 0], q["reward"], q["done"])
        for i in range(B):
            if self.batched_priorities:
                td_error = td[i]
            else:
                td_error = self.agent.get_td_error(state=q["state"][i], previous_action=q["previous_action"][i],
                                                   action=q["action"][i], reward=q["reward"][i], done=q["done"][i],
                                                   h=q["previous_h"][i], c=q["previous_c"][i])
            self.memory.add(td_error, [q[f][i] for f in FIELDS])

    def train(self):
        self.train_step += 1
        minibatch, idxs, weight = self.memory.sample(B)
        batch_state, batch_previous_action, batch_action = [], [], []
        batch_reward, batch_done, batch_previous_h, batch_previous_c = [], [], [], []
        for b in minibatch:
            batch_state.append(b[0])
            batch_previous_action.append(b[1])
            batch_action.append(b[2])
            batch_reward.append(b[3])
            batch_done.append(b[4])
            batch_previous_h.append(b[5])
            batch_previous_c.append(b[6])
        loss, td_error = self.agent.train(state=batch_state, previous_action=batch_previous_action,
                                          action=batch_action, h=batch_previous_h, c=batch_previous_c,
                                          reward=batch_reward, done=batch_done, weight=weight)
        for i in range(len(idxs)):
            self.memory.update(idxs[i], td_error[i])
        if self.train_step % TARGET_EVERY == 0:
            self.agent.main_to_target()
        return loss, list(idxs)


class DeviceArm:
    """The same loop on DeviceMemory + Agent.train_from_memory."""

    def __init__(self, agent, capacity, pool, errors):
        self.agent, self.train_step = agent, 0
        agent._get_engine(B)
        self.memory = agent.device_memory(capacity)
        arrs = [pool[f] for f in ("state", "previous_action", "action")] + \
            [pool["previous_h"][:, 0], pool["previous_c"][:, 0], pool["reward"], pool["done"]]
        for lo in range(0, len(errors), POOL):
            hi = min(lo + POOL, len(errors))
            self.memory.replay.add(None, *[a[:hi - lo] for a in arrs], error=errors[lo:hi])

    def ingest(self, q):
        self.memory.add(q["state"], q["previous_action"], q["action"], q["previous_h"], q["previous_c"], q["reward"],
                        q["done"])

    def train(self):
        self.train_step += 1
        loss, td_error = self.agent.train_from_memory(self.memory, B)
        if self.train_step % TARGET_EVERY == 0:
            self.agent.main_to_target()
        return loss, None

    def idxs(self):
        return self.memory.last_sample()[0].tolist()


def timed(arm, pool, k0, iters):
    ing, tr = [], []
    for k in range(k0, k0 + iters):
        q = queued(pool, k)
        t0 = time.perf_counter()
        arm.ingest(q)
        t1 = time.perf_counter()
        arm.train()
        t2 = time.perf_counter()
        ing.append(t1 - t0)
        tr.append(t2 - t1)
    return ing, tr


REPLAY_KERNELS = ("replay_sample_kernel", "replay_gather_seq_kernel", "replay_tree_update_kernel",
                  "replay_store_seq_kernel")


def profile(arm, pool, k0, iters, out_dir, name):
    """Kernels / copies per iteration and device time per replay kernel, from torch.profiler (its own run)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(k0, k0 + iters):
            arm.ingest(queued(pool, k))
            arm.train()
        torch.cuda.synchronize()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "r2d2_replay_%s.json" % name))
    kernels, copies, per = 0, 0, {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        nm = e.name
        if nm.startswith("Memcpy") or nm.startswith("Memset"):
            copies += 1
            continue
        kernels += 1
        for key in REPLAY_KERNELS:
            if key in nm:
                per.setdefault(key, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    return dict(kernels_per_iter=kernels / iters, copies_per_iter=copies / iters,
                replay_kernel_us={k: dict(median=float(np.median(v)), calls_per_iter=len(v) / iters)
                                  for k, v in sorted(per.items())})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=100000)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--iters", type=int, default=30, help="iterations per arm per round")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--parity", type=int, default=20, help="K: iterations compared from the same seeds")
    ap.add_argument("--graph", type=int, default=1)
    ap.add_argument("--profile-iters", type=int, default=10)
    ap.add_argument("--trace-dir", default=None, help="also write the profiler's chrome traces here")
    args = ap.parse_args()
    from distributed_reinforcement_learning_b200 import _native
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    if _native.device_count() < 1:
        raise SystemExit("bench_r2d2_replay needs a CUDA device (no CPU fallback)")
    info = gpu_info()
    pool = make_pool(0)
    kw = dict(num_action=A, lstm_size=L, input_shape=SHAPE)
    params = (r2d2_lstm.init_params(1, **kw), r2d2_lstm.init_params(2, **kw))
    errors = np.random.default_rng(3).exponential(1.0, args.capacity)
    g = bool(args.graph)
    host = HostArm(make_agent("bench_r2d2_host", params, g), args.capacity, pool, errors)
    dev = DeviceArm(make_agent("bench_r2d2_device", params, g), args.capacity, pool, errors)

    # parity: the first K iterations from the same seeds, parameters and memory contents; the host arm takes its
    # priorities from the learner's batched |td| (the per-sequence calls differ from it in float32 rounding)
    host.batched_priorities = True
    random.seed(123)
    hl, hi = [], []
    for k in range(args.parity):
        host.ingest(queued(pool, k))
        loss, idx = host.train()
        hl.append(loss)
        hi.append(idx)
    host.batched_priorities = False
    random.seed(123)
    dl, di = [], []
    for k in range(args.parity):
        dev.ingest(queued(pool, k))
        loss, _ = dev.train()
        dl.append(loss)
        di.append(dev.idxs())
    hl, dl = np.array(hl, np.float64), np.array(dl, np.float64)
    parity = dict(iterations=args.parity, same_indices=hi == di,
                  max_rel_loss_diff=float(np.max(np.abs(dl - hl) / np.maximum(np.abs(hl), 1e-30))))

    k = args.parity
    for arm in (host, dev):
        timed(arm, pool, k, args.warmup)
    k += args.warmup
    res = {"host": ([], []), "device": ([], [])}
    for _ in range(args.rounds):
        for name, arm in (("host", host), ("device", dev)):
            i, t = timed(arm, pool, k, args.iters)
            res[name][0].extend(i)
            res[name][1].extend(t)
        k += args.iters
    arms = {}
    for name, (i, t) in res.items():
        it = np.array(i) + np.array(t)
        arms[name] = dict(iter_ms=float(np.median(it)) * 1e3, iter_ms_p10=float(np.percentile(it, 10)) * 1e3,
                          iter_ms_p90=float(np.percentile(it, 90)) * 1e3, ingest_ms=float(np.median(i)) * 1e3,
                          train_ms=float(np.median(t)) * 1e3, sequences_per_s=B / float(np.median(it)),
                          iterations=len(it))
    eng = dev.agent._engine
    arms["learner_launches_per_step"] = eng.launches_per_step() if hasattr(eng, "launches_per_step") else None
    prof = {}
    try:
        for name, arm in (("host", host), ("device", dev)):
            prof[name] = profile(arm, pool, k, args.profile_iters, args.trace_dir, name)
            k += args.profile_iters
    except Exception as e:   # pragma: no cover - the profiler is optional
        prof = dict(error="not measured (%s)" % e)
    print(json.dumps(dict(bench="r2d2_replay", batch=B, seq_len=S, burn_in=BURN_IN, channels=SHAPE[-1], num_action=A,
                          capacity=args.capacity, use_cuda_graph=g, **info, parity=parity, arms=arms, profile=prof,
                          speedup=arms["host"]["iter_ms"] / arms["device"]["iter_ms"])))


if __name__ == "__main__":
    main()
