"""Environments in worker processes behind the policy server against VectorActor (`python tools/bench_actor_server.py`),
one GPU, one JSON line per per-step environment cost.

Both arms feed one DeviceFIFOQueue that impala.Agent.train_from_queue trains from, in one process, alternating blocks
of `--steps` learner steps:
  vector  VectorActor over n environments in the learner's thread (one unroll, then every learner step the queue
          holds a batch for)
  server  EnvWorkerPool of P spawned workers x k environments (P k = n), PolicyServer.run in a thread, the learner
          loop in the main thread
The environments are seeded synthetic ones (frames from a fixed pool) that spin for `--step-us` microseconds of host
work per step, to stand in for an emulator and its wrappers without ALE.  T = 20, A = 18, B = 32, lstm 256, CUDA
graphs on.  Reported per arm: environment frames/s and learner steps/s (median and min-max over blocks); for the
server the distribution of served batch sizes and, from a separate torch.profiler run, the mean device time of its
three kernels; H2D bytes per environment step computed from shapes; the card's name and power limit.

With `--family r2d2` the same comparison for R2D2 (`python tools/bench_actor_server.py --family r2d2`): both arms feed
one R2D2DeviceFIFOQueue, and one learner step is DeviceMemory.add_from_queue of a batch + Agent.train_from_memory, in
the main thread:
  vector  R2D2VectorActor over n environments in the learner's thread (one unroll of S steps, then every learner step
          the queue holds a batch for)
  server  R2D2EnvWorkerPool of P workers x k environments, R2D2PolicyServer.run in a thread
S = 15, burn-in 7, 84x84x1 frames, A = 4, B = 16, lstm 64, a replay memory filled with 4 batches before the timed
blocks, CUDA graphs on.

With `--family a3c` the same comparison for A3C (`python tools/bench_actor_server.py --family a3c --steps 64`): both
arms feed one A3CDeviceFIFOQueue, and one learner step is a3c.Agent.train_from_queue of one unroll, in the main thread:
  vector  A3CVectorActor over n environments in the learner's thread (one unroll of T steps, then every learner step
          the queue holds a record for)
  server  A3CEnvWorkerPool of P workers x k environments, A3CPolicyServer.run in a thread
T = 32, A = 4, a queue of 4n records, CUDA graphs on.  Environment frames/s and learner steps/s are reported as the
median and the 10th-90th percentiles over blocks.
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

T, A, L, B = 20, 18, 256, 32
SHAPE = (84, 84, 4)
FRAME = 84 * 84 * 4
VECTOR_H2D = FRAME + 4 + 4 * L + 4 * L + 8 + 5          # act row (frame, pa, h, c, uniform) + reward, done at commit
SERVER_REPORT_READ = FRAME + 4 * 16                     # frame + one 16-byte read per scalar report field

# the R2D2 family
R2_S, R2_BURN_IN, R2_A, R2_L, R2_B = 15, 7, 4, 64, 16
R2_SHAPE = (84, 84, 1)
R2_FRAME = 84 * 84 * 1
R2_VECTOR_H2D = R2_FRAME + 4 + 4 * R2_L + 4 * R2_L + 4 + 5   # act row (frame, pa, h, c, explore) + reward, done at commit
R2_SERVER_REPORT_READ = R2_FRAME + 3 * 16 + 4          # frame + 16-byte reads of reward, done, reset + the host's explore


# the A3C family
A3_T, A3_A = 32, 4
A3_VECTOR_H2D = FRAME + 4 + 8 + 4 + 1 + FRAME / A3_T   # act row (frame, pa, uniform) + reward, done and 1/T of the final
                                                       # next_state frame at commit (episode-reset frames not counted)
A3_SERVER_REPORT_READ = FRAME + 4 * 16                # frame + 16-byte reads of uniform, reward, done, reset (the
                                                       # next_state frame after an episode end not counted)


class BusyEnv:
    """Seeded synthetic environment: frames from a pool of 64, rewards in {0, 1}, a life lost now and then, episodes
    of up to 400 steps; every step spins for step_us microseconds."""

    def __init__(self, seed, step_us, shape=SHAPE):
        self.rng = np.random.RandomState(seed)
        self.step_us = step_us
        self.pool = np.random.default_rng(0).integers(0, 256, (64,) + tuple(shape), dtype=np.uint8)

    def reset(self):
        self.lives, self.t = 5, 0
        return self.pool[self.rng.randint(64)]

    def step(self, a):
        end = time.perf_counter() + self.step_us * 1e-6
        while time.perf_counter() < end:
            pass
        self.t += 1
        if self.rng.rand() < 0.01:
            self.lives -= 1
        done = self.lives == 0 or self.t >= 400
        return self.pool[self.rng.randint(64)], float(self.rng.rand() < 0.1), done, {"ale.lives": self.lives}


def make_env(seed, step_us, shape=SHAPE):
    return BusyEnv(seed, step_us, shape)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # pragma: no cover - informational only
        return dict(gpu="unknown (%s)" % e)


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


class VectorArm:
    def __init__(self, n, step_us, params):
        from distributed_reinforcement_learning_b200.actor import VectorActor
        from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
        from distributed_reinforcement_learning_b200.policy import NativePolicy
        self.agent = make_agent("bench_vector_%d" % step_us, params)
        self.queue = DeviceFIFOQueue(T, SHAPE, A, 4 * B, B, n, L)
        self.policy = NativePolicy(64, num_action=A)
        self.actor = VectorActor(self.policy, [make_env(i, step_us) for i in range(n)], self.queue, T, [A] * n,
                                 learner=self.agent)
        self.n = n

    def block(self, steps):
        t0, frames, done = time.perf_counter(), 0, 0
        while done < steps:
            self.actor.run_unroll()
            frames += self.n * T
            while self.queue.get_size() >= B and done < steps:
                self.agent.train_from_queue(self.queue)
                done += 1
        dt = time.perf_counter() - t0
        return frames / dt, steps / dt

    def close(self):
        self.policy.close()
        self.queue.close()


class ServerArm:
    def __init__(self, n, workers, step_us, params):
        import functools
        from distributed_reinforcement_learning_b200.actor_server import EnvWorkerPool, PolicyServer
        from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
        from distributed_reinforcement_learning_b200.policy import NativePolicy
        self.agent = make_agent("bench_server_%d" % step_us, params)
        self.queue = DeviceFIFOQueue(T, SHAPE, A, 4 * B, B, n, L)
        self.policy = NativePolicy(64, num_action=A)
        self.pool = EnvWorkerPool([functools.partial(make_env, i, step_us) for i in range(n)], [A] * n,
                                  n // workers, seeds=range(n))
        self.server = PolicyServer(self.policy, self.queue, self.pool, learner=self.agent)
        self.errors = []

    def _run(self, stop):
        try:
            self.server.run(stop)
        except Exception as e:   # pragma: no cover - reported by block()
            self.errors.append(e)

    def served(self):
        return sum(k * v for k, v in self.server.batch_sizes.items())

    def block(self, steps):
        """`steps` learner steps with the server running; it runs only inside blocks, and the batches it queued
        before one are trained first, untimed."""
        while self.queue.get_size() >= B:
            self.agent.train_from_queue(self.queue)
        stop = threading.Event()
        th = threading.Thread(target=self._run, args=(stop,))
        t0, f0 = time.perf_counter(), self.served()
        th.start()
        try:
            for _ in range(steps):
                self.agent.train_from_queue(self.queue, timeout_ms=300000)
            dt = time.perf_counter() - t0
            frames = self.served() - f0
        finally:
            stop.set()
            th.join()
        if self.errors:
            raise self.errors[0]
        return frames / dt, steps / dt

    def close(self):
        self.server.close()
        self.pool.close()
        self.policy.close()
        self.queue.close()


def server_kernel_ms(arm, steps, names=("server_gather_kernel", "queue_commit_rows_kernel", "server_scatter_kernel")):
    """Mean device time per launch of the server's kernels over `steps` learner steps (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm.block(steps)
        torch.cuda.synchronize()
    acc = {k: [] for k in names}
    for e in prof.events():
        for k in names:
            if k in e.name:
                acc[k].append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
    return {k: dict(launches=len(v), mean_us=float(np.mean(v)) if v else None) for k, v in acc.items()}


def stats(v):
    return dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))


def run(n, workers, step_us, blocks, steps, profile_steps, seed):
    from distributed_reinforcement_learning_b200.model import impala_actor_critic
    params = impala_actor_critic.init_params(seed=seed, num_action=A, lstm_hidden_size=L, input_shape=SHAPE)
    arms = dict(vector=VectorArm(n, step_us, params), server=ServerArm(n, workers, step_us, params))
    res = {k: dict(frames=[], steps=[]) for k in arms}
    try:
        for arm in arms.values():     # warm-up: graphs of every batch size met so far, the learner's first steps
            arm.block(2)
        sizes0 = dict(arms["server"].server.batch_sizes)
        for _ in range(blocks):
            for kind, arm in arms.items():
                f, s = arm.block(steps)
                res[kind]["frames"].append(f)
                res[kind]["steps"].append(s)
        sizes = {k: v - sizes0.get(k, 0) for k, v in sorted(arms["server"].server.batch_sizes.items())}
        kernels = server_kernel_ms(arms["server"], profile_steps) if profile_steps else None
    finally:
        for arm in arms.values():
            arm.close()
    words = 4 * (64 + 1 + 3 * 64)
    served = sum(k * v for k, v in sizes.items())
    serves = sum(sizes.values())
    out = dict(bench="actor_server", n=n, workers=workers, envs_per_worker=n // workers, step_us=step_us,
               trajectory=T, num_action=A, batch=B, blocks=blocks, learner_steps_per_block=steps)
    for kind in arms:
        out[kind] = dict(env_frames_per_s=stats(res[kind]["frames"]), learner_steps_per_s=stats(res[kind]["steps"]))
    out["vector"]["h2d_bytes_per_env_step"] = VECTOR_H2D
    out["server"].update(batch_sizes={str(k): v for k, v in sizes.items() if v},
                         mean_batch=served / serves if serves else None,
                         h2d_bytes_per_env_step=SERVER_REPORT_READ + (words * serves / served if served else 0),
                         kernels=kernels)
    out.update(gpu_info())
    return out


def make_r2d2_agent(name, params):
    from distributed_reinforcement_learning_b200.agent import r2d2
    ag = r2d2.Agent(R2_S, R2_BURN_IN, list(R2_SHAPE), R2_A, R2_L, 0.997, 1e-4, 1e-4, 1e9, 40.0, name, name)
    ag.use_cuda_graph = True
    ag._ensure_init()
    ag._main = params.copy()
    return ag


def r2d2_queue(n):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    return R2D2DeviceFIFOQueue(R2_S, R2_SHAPE, R2_A, 8 * R2_B, R2_B, n, R2_L)


class R2D2VectorArm:
    def __init__(self, n, step_us, params):
        from distributed_reinforcement_learning_b200.actor import R2D2VectorActor
        from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
        self.agent = make_r2d2_agent("bench_r2d2_vector_%d" % step_us, params)
        self.memory = self.agent.device_memory(1024)
        self.queue = r2d2_queue(n)
        self.policy = NativeR2D2Policy(64, num_action=R2_A, input_shape=R2_SHAPE)
        self.actor = R2D2VectorActor(self.policy, [make_env(i, step_us, R2_SHAPE) for i in range(n)], self.queue,
                                     R2_S, learner=self.agent)
        self.n = n

    def learner_step(self, timeout_ms=-1):
        self.memory.add_from_queue(self.queue, timeout_ms)
        self.agent.train_from_memory(self.memory, R2_B)

    def block(self, steps):
        t0, frames, done = time.perf_counter(), 0, 0
        while done < steps:
            self.actor.run_unroll()
            frames += self.n * R2_S
            while self.queue.get_size() >= R2_B and done < steps:
                self.learner_step()
                done += 1
        dt = time.perf_counter() - t0
        return frames / dt, steps / dt

    def close(self):
        self.policy.close()
        self.memory.close()
        self.queue.close()


class R2D2ServerArm(ServerArm):
    def __init__(self, n, workers, step_us, params):
        import functools
        from distributed_reinforcement_learning_b200.actor_server import R2D2EnvWorkerPool, R2D2PolicyServer
        from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy
        self.agent = make_r2d2_agent("bench_r2d2_server_%d" % step_us, params)
        self.memory = self.agent.device_memory(1024)
        self.queue = r2d2_queue(n)
        self.policy = NativeR2D2Policy(64, num_action=R2_A, input_shape=R2_SHAPE)
        self.pool = R2D2EnvWorkerPool([functools.partial(make_env, i, step_us, R2_SHAPE) for i in range(n)], R2_A,
                                      n // workers, seeds=range(n))
        self.server = R2D2PolicyServer(self.policy, self.queue, self.pool, learner=self.agent)
        self.errors = []

    def learner_step(self, timeout_ms=-1):
        self.memory.add_from_queue(self.queue, timeout_ms)
        self.agent.train_from_memory(self.memory, R2_B)

    def block(self, steps):
        """`steps` learner steps with the server running; it runs only inside blocks, and the batches it queued
        before one are ingested and trained first, untimed."""
        while self.queue.get_size() >= R2_B:
            self.learner_step()
        stop = threading.Event()
        th = threading.Thread(target=self._run, args=(stop,))
        t0, f0 = time.perf_counter(), self.served()
        th.start()
        try:
            for _ in range(steps):
                self.learner_step(timeout_ms=300000)
            dt = time.perf_counter() - t0
            frames = self.served() - f0
        finally:
            stop.set()
            th.join()
        if self.errors:
            raise self.errors[0]
        return frames / dt, steps / dt

    def close(self):
        super().close()
        self.memory.close()


def run_r2d2(n, workers, step_us, blocks, steps, profile_steps, seed):
    from distributed_reinforcement_learning_b200.model import r2d2_lstm
    params = r2d2_lstm.init_params(seed, num_action=R2_A, lstm_size=R2_L, input_shape=R2_SHAPE)
    arms = dict(vector=R2D2VectorArm(n, step_us, params), server=R2D2ServerArm(n, workers, step_us, params))
    res = {k: dict(frames=[], steps=[]) for k in arms}
    try:
        for arm in arms.values():     # warm-up: graphs of every batch size met so far; fills the memory with 4 batches
            arm.block(4)
        sizes0 = dict(arms["server"].server.batch_sizes)
        for _ in range(blocks):
            for kind, arm in arms.items():
                f, s = arm.block(steps)
                res[kind]["frames"].append(f)
                res[kind]["steps"].append(s)
        sizes = {k: v - sizes0.get(k, 0) for k, v in sorted(arms["server"].server.batch_sizes.items())}
        names = ("r2d2_server_gather_kernel", "queue_commit_rows_kernel", "r2d2_server_scatter_kernel")
        kernels = server_kernel_ms(arms["server"], profile_steps, names) if profile_steps else None
    finally:
        for arm in arms.values():
            arm.close()
    words = 4 * (64 + 1 + 3 * 64 + 64)
    served = sum(k * v for k, v in sizes.items())
    serves = sum(sizes.values())
    out = dict(bench="actor_server_r2d2", n=n, workers=workers, envs_per_worker=n // workers, step_us=step_us,
               seq_len=R2_S, burn_in=R2_BURN_IN, num_action=R2_A, batch=R2_B, blocks=blocks,
               learner_steps_per_block=steps)
    for kind in arms:
        out[kind] = dict(env_frames_per_s=stats(res[kind]["frames"]), learner_steps_per_s=stats(res[kind]["steps"]))
    out["vector"]["h2d_bytes_per_env_step"] = R2_VECTOR_H2D
    out["server"].update(batch_sizes={str(k): v for k, v in sizes.items() if v},
                         mean_batch=served / serves if serves else None,
                         h2d_bytes_per_env_step=R2_SERVER_REPORT_READ + (words * serves / served if served else 0),
                         kernels=kernels)
    out.update(gpu_info())
    return out


def pstats(v):
    return dict(median=float(np.median(v)), p10=float(np.percentile(v, 10)), p90=float(np.percentile(v, 90)))


def make_a3c_agent(name, params):
    from distributed_reinforcement_learning_b200.agent import a3c
    ag = a3c.Agent(SHAPE, A3_A, 0.99, 1e-4, 0.0, 1e9, 0.5, 0.01, 40.0, "abs_one", name, name)
    ag.use_cuda_graph = True
    ag._ensure_init()
    ag._params = params.copy()
    ag._get_engine(A3_T)
    return ag


def a3c_queue(n):
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    return A3CDeviceFIFOQueue(A3_T, SHAPE, A3_A, n, queue_size=4 * n)


class A3CVectorArm:
    def __init__(self, n, step_us, params):
        from distributed_reinforcement_learning_b200.actor import A3CVectorActor
        from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
        self.agent = make_a3c_agent("bench_a3c_vector_%d" % step_us, params)
        self.queue = a3c_queue(n)
        self.policy = NativeA3CPolicy(64, num_action=A3_A, input_shape=SHAPE)
        self.actor = A3CVectorActor(self.policy, [make_env(i, step_us) for i in range(n)], self.queue, A3_T,
                                    [A3_A] * n, learner=self.agent)
        self.n = n

    def block(self, steps):
        t0, frames, done = time.perf_counter(), 0, 0
        while done < steps:
            self.actor.run_unroll()
            frames += self.n * A3_T
            while self.queue.get_size() >= 1 and done < steps:
                self.agent.train_from_queue(self.queue)
                done += 1
        dt = time.perf_counter() - t0
        return frames / dt, steps / dt

    def close(self):
        self.policy.close()
        self.queue.close()


class A3CServerArm(ServerArm):
    def __init__(self, n, workers, step_us, params):
        import functools
        from distributed_reinforcement_learning_b200.actor_server import A3CEnvWorkerPool, A3CPolicyServer
        from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
        self.agent = make_a3c_agent("bench_a3c_server_%d" % step_us, params)
        self.queue = a3c_queue(n)
        self.policy = NativeA3CPolicy(64, num_action=A3_A, input_shape=SHAPE)
        self.pool = A3CEnvWorkerPool([functools.partial(make_env, i, step_us) for i in range(n)], [A3_A] * n,
                                     n // workers, seeds=range(n))
        self.server = A3CPolicyServer(self.policy, self.queue, self.pool, learner=self.agent)
        self.errors = []

    def block(self, steps):
        """`steps` learner steps with the server running; it runs only inside blocks, and the records it queued
        before one are trained on first, untimed."""
        while self.queue.get_size() >= 1:
            self.agent.train_from_queue(self.queue)
        stop = threading.Event()
        th = threading.Thread(target=self._run, args=(stop,))
        t0, f0 = time.perf_counter(), self.served()
        th.start()
        try:
            for _ in range(steps):
                self.agent.train_from_queue(self.queue, timeout_ms=300000)
            dt = time.perf_counter() - t0
            frames = self.served() - f0
        finally:
            stop.set()
            th.join()
        if self.errors:
            raise self.errors[0]
        return frames / dt, steps / dt


def run_a3c(n, workers, step_us, blocks, steps, profile_steps, seed):
    from distributed_reinforcement_learning_b200.model import actor_critic
    params = actor_critic.init_params(seed, num_action=A3_A, input_shape=SHAPE)
    arms = dict(vector=A3CVectorArm(n, step_us, params), server=A3CServerArm(n, workers, step_us, params))
    res = {k: dict(frames=[], steps=[]) for k in arms}
    try:
        for arm in arms.values():     # warm-up: graphs of every batch size met so far, the learner's first steps
            arm.block(2)
        sizes0 = dict(arms["server"].server.batch_sizes)
        for _ in range(blocks):
            for kind, arm in arms.items():
                f, s = arm.block(steps)
                res[kind]["frames"].append(f)
                res[kind]["steps"].append(s)
        sizes = {k: v - sizes0.get(k, 0) for k, v in sorted(arms["server"].server.batch_sizes.items())}
        names = ("a3c_server_gather_kernel", "queue_commit_rows_kernel", "a3c_server_scatter_kernel")
        kernels = server_kernel_ms(arms["server"], profile_steps, names) if profile_steps else None
    finally:
        for arm in arms.values():
            arm.close()
    words = 4 * (64 + 1 + 3 * 64)
    served = sum(k * v for k, v in sizes.items())
    serves = sum(sizes.values())
    out = dict(bench="actor_server_a3c", n=n, workers=workers, envs_per_worker=n // workers, step_us=step_us,
               trajectory=A3_T, num_action=A3_A, blocks=blocks, learner_steps_per_block=steps)
    for kind in arms:
        out[kind] = dict(env_frames_per_s=pstats(res[kind]["frames"]),
                         learner_steps_per_s=pstats(res[kind]["steps"]))
    out["vector"]["h2d_bytes_per_env_step"] = A3_VECTOR_H2D
    out["server"].update(batch_sizes={str(k): v for k, v in sizes.items() if v},
                         mean_batch=served / serves if serves else None,
                         h2d_bytes_per_env_step=A3_SERVER_REPORT_READ + (words * serves / served if served else 0),
                         kernels=kernels)
    out.update(gpu_info())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--family", choices=("impala", "r2d2", "a3c"), default="impala")
    ap.add_argument("--n", type=int, default=32, help="environments")
    ap.add_argument("--workers", type=int, default=8, help="worker processes P (n / P environments each)")
    ap.add_argument("--step-us", default="0,200,1000", help="host work per environment step, microseconds")
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10, help="learner steps per block")
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    if a.n % a.workers:
        raise SystemExit("--n must be a multiple of --workers")
    from distributed_reinforcement_learning_b200 import _native as N
    if N.device_count() < 1:
        raise SystemExit("needs a CUDA device (no CPU fallback)")
    bench = dict(impala=run, r2d2=run_r2d2, a3c=run_a3c)[a.family]
    for us in [int(x) for x in a.step_us.split(",")]:
        print(json.dumps(bench(a.n, a.workers, us, a.blocks, a.steps, a.profile_steps, a.seed)), flush=True)


if __name__ == "__main__":
    main()
