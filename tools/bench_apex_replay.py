"""The Ape-X learner loop with the replay memory on the host and on the GPU (`python tools/bench_apex_replay.py`), one
H100, one JSON line.

Both arms run the learner branch of train_apex.py:82-155 at the reference configuration (batch 32, trajectory 32,
num_action 4, capacity 1e5 pre-filled) in the same process, alternating blocks of iterations:
  host    apex.Agent + buffer_queue.Memory, the loop as the reference writes it: get_td_error, 32 Memory.add, then
          Memory.sample, np.array + six np.stack, distributed_train, 32 Memory.update
  device  apex.Agent.device_memory + DeviceMemory.add (ingest) + Agent.train_from_memory (train)
One iteration = one actor record of 32 transitions ingested + one training step.  The memory is filled, and the records
drawn, from a pool of 1,024 distinct synthetic transitions (the host arm stores views of the pool's arrays).
Reported per arm: wall ms per iteration (median), its ingest / train split, transitions trained per second (32 per
iteration), and from a separate torch.profiler run of a few iterations the kernels and copies per iteration and the
device time of the replay kernels (sample, gather, tree update, store).  The device arm's ingest only enqueues work;
its device time lands in the train call that follows, so only the sum is comparable.  Also: for the first K
iterations from the same seeds and the same parameters, whether both arms sampled the same indices, and the largest
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

A, B, TRAJ, POOL = 4, 32, 32, 1024
SHAPE = (84, 84, 4)


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
    return dict(state=rng.integers(0, 256, (POOL,) + SHAPE, dtype=np.uint8),
                next_state=rng.integers(0, 256, (POOL,) + SHAPE, dtype=np.uint8),
                previous_action=rng.integers(0, A, POOL).astype(np.int32),
                action=rng.integers(0, A, POOL).astype(np.int32),
                reward=(rng.standard_normal(POOL) * 2).astype(np.float32), done=rng.random(POOL) < 0.1)


FIELDS = ("state", "next_state", "previous_action", "action", "reward", "done")


def record(pool, k):
    lo = (k * TRAJ) % POOL
    return tuple(pool[f][lo:lo + TRAJ] for f in FIELDS)


def make_agent(name, params, graph):
    from distributed_reinforcement_learning_b200.agent import apex
    a = apex.Agent(input_shape=SHAPE, num_action=A, discount_factor=0.99, gradient_clip_norm=40.0,
                   reward_clipping="abs_one", start_learning_rate=1e-4, end_learning_rate=0.0,
                   learning_frame=100000000000000, model_name=name, learner_name=name)
    a.use_cuda_graph = graph
    a._main, a._target = params[0].copy(), params[1].copy()
    z = np.zeros_like(a._main)
    a._opt = dict(m=z, v=z.copy(), step=0, beta1_power=0.9, beta2_power=0.999)
    a.target_to_main()
    return a


class HostArm:
    """train_apex.py:82-155 as written, on apex.Agent + buffer_queue.Memory."""

    def __init__(self, agent, capacity, pool, errors):
        from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import Memory
        self.agent, self.memory, self.train_step = agent, Memory(capacity), 0
        for i, e in enumerate(errors):
            j = i % POOL
            self.memory.add(e, [pool[f][j] for f in FIELDS])

    def ingest(self, rec):
        st, ns, pa, ac, rw, dn = rec
        td_error = self.agent.get_td_error(state=st, next_state=ns, previous_action=pa, action=ac, reward=rw, done=dn)
        for i in range(len(td_error)):
            self.memory.add(td_error[i], [st[i], ns[i], pa[i], ac[i], rw[i], dn[i]])

    def train(self):
        self.train_step += 1
        minibatch, idxs, is_weight = self.memory.sample(B)
        minibatch = np.array(minibatch, dtype=object)
        loss, td_error = self.agent.distributed_train(
            state=np.stack(minibatch[:, 0]), next_state=np.stack(minibatch[:, 1]),
            previous_action=np.stack(minibatch[:, 2]), action=np.stack(minibatch[:, 3]),
            reward=np.stack(minibatch[:, 4]), done=np.stack(minibatch[:, 5]), is_weight=is_weight)
        if self.train_step % 100 == 0:
            self.agent.target_to_main()
        for i in range(len(idxs)):
            self.memory.update(idxs[i], td_error[i])
        return loss, list(idxs)


class DeviceArm:
    """The same loop on DeviceMemory + Agent.train_from_memory."""

    def __init__(self, agent, capacity, pool, errors):
        self.agent, self.train_step = agent, 0
        self.memory = agent.device_memory(capacity)
        arrs = [pool[f] for f in FIELDS]
        for lo in range(0, len(errors), POOL):
            hi = min(lo + POOL, len(errors))
            self.memory.replay.add(None, *[a[:hi - lo] for a in arrs], error=errors[lo:hi])

    def ingest(self, rec):
        self.memory.add(*rec)

    def train(self):
        self.train_step += 1
        loss, td_error = self.agent.train_from_memory(self.memory, B)
        if self.train_step % 100 == 0:
            self.agent.target_to_main()
        return loss, None

    def idxs(self):
        return self.memory.last_sample()[0].tolist()


def timed(arm, pool, k0, iters):
    ing, tr = [], []
    for k in range(k0, k0 + iters):
        rec = record(pool, k)
        t0 = time.perf_counter()
        arm.ingest(rec)
        t1 = time.perf_counter()
        arm.train()
        t2 = time.perf_counter()
        ing.append(t1 - t0)
        tr.append(t2 - t1)
    return ing, tr


def profile(arm, pool, k0, iters, out_dir, name):
    """Kernels / copies per iteration and device time per replay kernel, from torch.profiler (its own run)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(k0, k0 + iters):
            arm.ingest(record(pool, k))
            arm.train()
        torch.cuda.synchronize()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "apex_replay_%s.json" % name))
    kernels, copies, per = 0, 0, {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        nm = e.name
        if nm.startswith("Memcpy") or nm.startswith("Memset"):
            copies += 1
            continue
        kernels += 1
        for key in ("replay_sample_kernel", "apex_replay_gather_kernel", "replay_tree_update_kernel",
                    "apex_replay_store_kernel"):
            if key in nm:
                per.setdefault(key, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    return dict(kernels_per_iter=kernels / iters, copies_per_iter=copies / iters,
                replay_kernel_us={k: dict(median=float(np.median(v)), calls_per_iter=len(v) / iters)
                                  for k, v in sorted(per.items())})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=100000)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--iters", type=int, default=50, help="iterations per arm per round")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--parity", type=int, default=20, help="K: iterations compared from the same seeds")
    ap.add_argument("--graph", type=int, default=1)
    ap.add_argument("--profile-iters", type=int, default=10)
    ap.add_argument("--trace-dir", default=None, help="also write the profiler's chrome traces here")
    args = ap.parse_args()
    from distributed_reinforcement_learning_b200 import _native
    from distributed_reinforcement_learning_b200.model import apex_value
    if _native.device_count() < 1:
        raise SystemExit("bench_apex_replay needs a CUDA device (no CPU fallback)")
    info = gpu_info()
    pool = make_pool(0)
    params = (apex_value.init_params(1, num_action=A, input_shape=SHAPE),
              apex_value.init_params(2, num_action=A, input_shape=SHAPE))
    errors = np.random.default_rng(3).exponential(1.0, args.capacity)
    g = bool(args.graph)
    host = HostArm(make_agent("bench_host", params, g), args.capacity, pool, errors)
    dev = DeviceArm(make_agent("bench_device", params, g), args.capacity, pool, errors)

    # parity: the first K iterations from the same seeds, parameters and memory contents
    random.seed(123)
    hl, hi = [], []
    for k in range(args.parity):
        host.ingest(record(pool, k))
        loss, idx = host.train()
        hl.append(loss)
        hi.append(idx)
    random.seed(123)
    dl, di = [], []
    for k in range(args.parity):
        dev.ingest(record(pool, k))
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
                          train_ms=float(np.median(t)) * 1e3, transitions_per_s=B / float(np.median(it)),
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
    print(json.dumps(dict(bench="apex_replay", batch=B, trajectory=TRAJ, num_action=A, capacity=args.capacity,
                          use_cuda_graph=g, **info, parity=parity, arms=arms, profile=prof,
                          speedup=arms["host"]["iter_ms"] / arms["device"]["iter_ms"])))


if __name__ == "__main__":
    main()
