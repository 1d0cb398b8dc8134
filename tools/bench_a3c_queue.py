"""The co-located A3C actor -> learner loop with the trajectory queue on the host and on the GPU
(`python tools/bench_a3c_queue.py`), one H100, one JSON line per actor count.

Both arms run the loop of train_a3c.py in one process, alternating blocks of iterations:
  host    A3CVectorActor + buffer_queue.A3CFIFOQueue: every appended unroll is sampled and trained on at once
          (Agent.train: np.stack of state and next_state, then drl_a3c_stage uploads the record)
  device  A3CVectorActor + buffer_queue.A3CDeviceFIFOQueue (the A3C recorder writes each step on the device, one commit
          per unroll) + n x Agent.train_from_queue (the record is staged device to device)
One iteration = one unroll of n environments (the learner's parameters synced into the policy first, T batched acts)
followed by n training steps, one per environment's unroll.  The environments are cheap seeded synthetic ones (frames
drawn from a fixed pool, an episode end every few hundred steps), so the loop measures the engine, the queue and the
learner, not an emulator.  T = 32, A = 4, 84x84x4 frames, CUDA graphs on (the reference's configuration otherwise).
Reported per arm: ms per iteration (median, p10-p90), actor and learner ms per iteration (medians), environment
frames per second, the H2D bytes per iteration computed from shapes (the acts' inputs, and what moves the records),
and the kernels and copies per iteration counted from the code paths.  The first K iterations of both arms start from
the same seeds and parameters; their losses and final parameters must be bit-equal (bit_equal).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

T, A = 32, 4
SHAPE = (84, 84, 4)
FRAME = 84 * 84 * 4
# one record as drl_a3c_stage uploads it: 2T frames, previous_action + action, reward, done and the unit weights
RECORD_H2D = 2 * T * FRAME + 2 * T * 4 + T * 4 + T + T * 4   # 1,806,880 B


def align(b):
    return -(-b // 256) * 256


def act_h2d(n):
    """One act's input block (apex_policy.cu: apex_in_layout): n frames, previous actions, uniforms."""
    return align(n * FRAME) + align(n * 4) + align(n * 8)


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
    episodes of a few hundred steps.  `uploads` counts the episode resets whose frame the next act has to upload (an
    episode that ends at the last step of an unroll hands its terminal frame to the commit instead)."""
    POOL = None

    def __init__(self, seed):
        if PoolEnv.POOL is None:
            PoolEnv.POOL = np.random.default_rng(0).integers(0, 256, (64,) + SHAPE, dtype=np.uint8)
        self.rng = np.random.RandomState(seed)
        self.steps, self.reset_steps = 0, []

    def reset(self):
        self.lives, self.t = 5, 0
        self.reset_steps.append(self.steps)
        return PoolEnv.POOL[self.rng.randint(64)]

    def step(self, a):
        self.t += 1
        self.steps += 1
        if self.rng.rand() < 0.01:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 400
        return PoolEnv.POOL[self.rng.randint(64)], float(self.rng.rand() < 0.1), done, {"ale.lives": self.lives}


def make_agent(name, params):
    from distributed_reinforcement_learning_b200.agent import a3c
    ag = a3c.Agent(list(SHAPE), A, 0.997, 1e-4, 0.0, 1e9, 0.5, 0.05, 40.0, "abs_one", name, name)
    ag.use_cuda_graph = True
    ag.set_session(None)
    ag._params = params.copy()
    ag._get_engine(T)
    return ag


class TrainingQueue:
    """A3CFIFOQueue with train_a3c.py's learner behind it: every appended unroll is sampled and trained on at once."""

    def __init__(self, queue, agent, out):
        self.queue, self.agent, self.out, self.train_s = queue, agent, out, 0.0

    def append_to_queue(self, **kw):
        t0 = time.perf_counter()
        self.queue.append_to_queue(**kw)
        b = self.queue.sample_batch()
        self.out.append(self.agent.train(state=b.state[0], next_state=b.next_state[0],
                                         previous_action=b.previous_action[0], action=b.action[0],
                                         reward=b.reward[0], done=b.done[0]))
        self.train_s += time.perf_counter() - t0


class Arm:
    def __init__(self, kind, n, params, seed):
        from distributed_reinforcement_learning_b200.actor import A3CVectorActor
        from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
        from distributed_reinforcement_learning_b200.distributed_queue import buffer_queue as bq
        self.kind, self.n = kind, n
        self.agent = make_agent("bench_a3cq_%s_%d" % (kind, n), params)
        self.out = []
        if kind == "host":
            self.queue = TrainingQueue(bq.A3CFIFOQueue(T, SHAPE, A, n), self.agent, self.out)
        else:
            self.queue = bq.A3CDeviceFIFOQueue(T, SHAPE, A, n)
        self.policy = NativeA3CPolicy(64, num_action=A, input_shape=SHAPE, use_cuda_graph=True)
        self.envs = [PoolEnv(seed * 1000 + i) for i in range(n)]
        self.actor = A3CVectorActor(self.policy, self.envs, self.queue, T, [A] * n, learner=self.agent)

    def iteration(self):
        """-> actor s, learner s, reset frames the device arm uploads in its acts."""
        marks = [(e.steps, len(e.reset_steps)) for e in self.envs]
        t0 = time.perf_counter()
        if self.kind == "host":
            self.queue.train_s = 0.0
            self.actor.run_unroll()
            tl = self.queue.train_s
            ta = time.perf_counter() - t0 - tl
        else:
            self.actor.run_unroll()
            t1 = time.perf_counter()
            for _ in range(self.n):
                self.out.append(self.agent.train_from_queue(self.queue))
            ta, tl = t1 - t0, time.perf_counter() - t1
        last = [s0 + T for s0, _ in marks]    # a reset after the unroll's last step feeds no act of this unroll
        uploads = sum(sum(1 for s in e.reset_steps[r0:] if s < last[i]) for i, (e, (_, r0)) in
                      enumerate(zip(self.envs, marks)))
        return ta, tl, uploads


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def run(n, blocks, iters, parity, seed):
    from distributed_reinforcement_learning_b200.model import actor_critic
    params = actor_critic.init_params(seed, num_action=A, input_shape=SHAPE)
    arms = {}
    for kind in ("host", "device"):
        np.random.seed(seed)
        arms[kind] = Arm(kind, n, params, seed)
        for _ in range(parity):
            arms[kind].iteration()
    h, d = arms["host"], arms["device"]
    bit_equal = len(h.out) == len(d.out) == n * parity and h.out == d.out and \
        np.array_equal(h.agent._engine.get_params(), d.agent._engine.get_params())
    steps_per_launch = h.agent._engine.launches_per_step() if hasattr(h.agent._engine, "launches_per_step") else None
    res = {k: dict(actor=[], learner=[], total=[], uploads=0, iters=0) for k in arms}
    for _ in range(blocks):
        for kind, arm in arms.items():
            r = res[kind]
            for _ in range(iters):
                ta, tl, up = arm.iteration()
                r["actor"].append(ta)
                r["learner"].append(tl)
                r["total"].append(ta + tl)
                r["uploads"] += up
                r["iters"] += 1
    out = {}
    for kind, r in res.items():
        acts = T * act_h2d(n)
        if kind == "host":
            record_h2d = n * RECORD_H2D
            # per act: 1 H2D + conv1/conv2/conv3/skinny_splitk/head; per record: drl_a3c_stage's 7 H2Ds
            kernels, copies = 5 * T, T + 7 * n
        else:
            # commit: reward + done (5 B per step) and the n final next_state frames; the acts' reset frames; the
            # stage's unit weights
            record_h2d = n * T * 5 + n * FRAME + r["uploads"] / r["iters"] * FRAME + n * T * 4
            # per act: 1 H2D + the 5 kernels + a3c_record_step; commit: 3 H2Ds + 4 D2Ds per record; stage: 4 D2Ds +
            # the weights' H2D
            kernels, copies = 6 * T, T + 3 + 4 * n + 5 * n
        total_s = float(np.sum(r["total"]))
        out[kind] = dict(
            ms_per_iter=pct(r["total"], 50), ms_p10=pct(r["total"], 10), ms_p90=pct(r["total"], 90),
            actor_ms=pct(r["actor"], 50), learner_ms=pct(r["learner"], 50),
            env_frames_per_s=n * T * r["iters"] / total_s,
            act_h2d_bytes_per_iter=acts, record_h2d_bytes_per_iter=int(record_h2d),
            reset_frames_per_iter=r["uploads"] / r["iters"] if kind == "device" else None,
            policy_kernels_per_iter=kernels, copies_per_iter_excl_learner_step=copies)
    return dict(bench="a3c_queue", n=n, trajectory=T, num_action=A, cuda_graph=True, blocks=blocks,
                iters_per_block=iters, parity_iters=parity, bit_equal=bool(bit_equal),
                learner_launches_per_step=steps_per_launch, host=out["host"], device=out["device"],
                ms_per_iter_speedup=out["host"]["ms_per_iter"] / out["device"]["ms_per_iter"], **gpu_info())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="1,20", help="environments per actor (comma-separated)")
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--iters", type=int, default=4, help="iterations per arm per block")
    ap.add_argument("--parity", type=int, default=2, help="K: iterations compared from the same seeds")
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
