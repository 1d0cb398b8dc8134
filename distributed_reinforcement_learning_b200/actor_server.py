"""IMPALA environments in worker processes, served by one batched policy engine beside the learner.

The reference runs every actor in its own process (``train_impala.py``); ``VectorActor`` steps all its environments
one after another in one thread.  Here the environments step in parallel in CPU-only worker processes
(``EnvWorkerPool``), and one ``PolicyServer`` in the learner's process acts for all of them through one
``NativePolicy`` (``drl_policy_server_*``, include/drl_b200.h), with every environment's h, c, previous action and
unfinished trajectory kept on the GPU.  Completed trajectories go into a ``DeviceFIFOQueue`` that
``impala.Agent.train_from_queue`` trains from.

Workers and server share one exchange block (``multiprocessing.shared_memory``): a report record per environment
(the frame to act on, the uniform draw of the action, the reward and done of the previous step, a reset flag) and a
reply record per environment (action, max probability), laid out as ``DRL_SERVER_*`` in include/drl_b200.h.  The
server registers the block with CUDA; its kernels read the reports and write the replies directly.  A worker writes
its environments' reports, then signals on its pipe; the server answers on the same pipe once the replies are written.

R2D2 has the same pair: ``R2D2EnvWorkerPool`` steps R2D2 environments under ``utils.r2d2_env_step`` and draws each
environment's explore decision from its own stream, and ``R2D2PolicyServer`` acts for them through one
``NativeR2D2Policy`` (``drl_r2d2_policy_server_*``) into an ``R2D2DeviceFIFOQueue`` that
``r2d2.DeviceMemory.add_from_queue`` ingests.  Its records (``DRL_R2D2_SERVER_*``) have the IMPALA records' sizes; the
report carries an explore action instead of a uniform draw, and the reply q_action instead of a max probability.

A3C has the pair ``A3CEnvWorkerPool`` / ``A3CPolicyServer``: the IMPALA step rule (``utils.impala_env_step``), one
``NativeA3CPolicy`` (``drl_a3c_policy_server_*``) and an ``A3CDeviceFIFOQueue`` that ``a3c.Agent.train_from_queue``
trains from.  An A3C record stores next_state, and after an episode end the frame to act on (the new episode's first)
is not the previous step's next_state, so its report (``DRL_A3C_SERVER_*``) carries a second frame, written and read
only then.

Ape-X has the pair ``ApexEnvWorkerPool`` / ``ApexPolicyServer``: the Ape-X step rule (``utils.apex_env_step``), one
``NativeApexPolicy`` (``drl_apex_policy_server_*``) and an ``ApexDeviceFIFOQueue`` that ``apex.DeviceMemory
.add_from_queue`` ingests.  Each environment's ``LocalBuffer`` is a ring on the GPU.  A worker keeps only a count of
its buffer's length and draws the sample order (``LocalBuffer.sample``'s permutation) itself, so its report
(``DRL_APEX_SERVER_*``) carries the explore action, the order and, after an episode end, the previous step's
next_state.

This module imports neither torch nor the native library at module level: the spawned workers import it.
"""
import collections
import ctypes as C
import multiprocessing as mp
import multiprocessing.connection
import pickle
import sys
import threading
import traceback
from multiprocessing import shared_memory

import numpy as np

from . import utils

# the exchange block's records (include/drl_b200.h: DRL_SERVER_*)
FRAME_SHAPE = (84, 84, 4)
REPORT_FRAME, REPORT_UNIFORM, REPORT_REWARD, REPORT_DONE, REPORT_RESET, REPORT_BYTES = 0, 28224, 28240, 28256, 28272, 28288
REPLY_ACTION, REPLY_MAX_PROB, REPLY_BYTES = 0, 16, 32
PAGE = 4096
MAX_ENVS = 256


def exchange_bytes(num_envs):
    """Size of the exchange block of num_envs environments: the reports, then the replies, rounded up to a page."""
    n = num_envs * (REPORT_BYTES + REPLY_BYTES)
    return -(-n // PAGE) * PAGE


def exchange_views(buf, num_envs):
    """numpy views of the records in the exchange block `buf` (a writable buffer of exchange_bytes(num_envs))."""
    E = num_envs

    def field(offset, dtype, shape=(), strides=()):
        return np.ndarray((E,) + shape, dtype, buffer=buf, offset=offset, strides=(stride,) + strides)

    stride = REPORT_BYTES
    v = dict(frame=field(REPORT_FRAME, np.uint8, FRAME_SHAPE, (FRAME_SHAPE[1] * FRAME_SHAPE[2], FRAME_SHAPE[2], 1)),
             uniform=field(REPORT_UNIFORM, np.float64), reward=field(REPORT_REWARD, np.float32),
             done=field(REPORT_DONE, np.uint8), reset=field(REPORT_RESET, np.uint8))
    stride = REPLY_BYTES
    base = E * REPORT_BYTES
    v.update(action=field(base + REPLY_ACTION, np.int32), max_prob=field(base + REPLY_MAX_PROB, np.float32))
    return v


# the R2D2 server's records (include/drl_b200.h: DRL_R2D2_SERVER_*): the IMPALA records' sizes and stride
R2D2_REPORT_FRAME, R2D2_REPORT_EXPLORE, R2D2_REPORT_REWARD, R2D2_REPORT_DONE, R2D2_REPORT_RESET, R2D2_REPORT_BYTES = (
    0, 28224, 28240, 28256, 28272, 28288)
R2D2_REPLY_ACTION, R2D2_REPLY_Q_ACTION, R2D2_REPLY_BYTES = 0, 16, 32


def r2d2_exchange_views(buf, num_envs, channels=1):
    """numpy views of the R2D2 records in the exchange block `buf` (a writable buffer of exchange_bytes(num_envs));
    frames are 84x84x`channels`."""
    E, shape = num_envs, (84, 84, int(channels))

    def field(offset, dtype, shape=(), strides=()):
        return np.ndarray((E,) + shape, dtype, buffer=buf, offset=offset, strides=(stride,) + strides)

    stride = R2D2_REPORT_BYTES
    v = dict(frame=field(R2D2_REPORT_FRAME, np.uint8, shape, (shape[1] * shape[2], shape[2], 1)),
             explore=field(R2D2_REPORT_EXPLORE, np.int32), reward=field(R2D2_REPORT_REWARD, np.float32),
             done=field(R2D2_REPORT_DONE, np.uint8), reset=field(R2D2_REPORT_RESET, np.uint8))
    stride = R2D2_REPLY_BYTES
    base = E * R2D2_REPORT_BYTES
    v.update(action=field(base + R2D2_REPLY_ACTION, np.int32), q_action=field(base + R2D2_REPLY_Q_ACTION, np.float32))
    return v


# the A3C server's records (include/drl_b200.h: DRL_A3C_SERVER_*): two frames per report
A3C_REPORT_FRAME, A3C_REPORT_NEXT_STATE, A3C_REPORT_UNIFORM, A3C_REPORT_REWARD, A3C_REPORT_DONE, A3C_REPORT_RESET = (
    0, 28224, 56448, 56464, 56480, 56496)
A3C_REPORT_BYTES = 56512
A3C_REPLY_ACTION, A3C_REPLY_MAX_PROB, A3C_REPLY_BYTES = 0, 16, 32


def a3c_exchange_bytes(num_envs):
    """Size of the A3C exchange block of num_envs environments: the reports, then the replies, rounded up to a page."""
    n = num_envs * (A3C_REPORT_BYTES + A3C_REPLY_BYTES)
    return -(-n // PAGE) * PAGE


def a3c_exchange_views(buf, num_envs):
    """numpy views of the A3C records in the exchange block `buf` (a writable buffer of a3c_exchange_bytes(num_envs)):
    frame, next_state, uniform, reward, done, reset, action and max_prob."""
    E = num_envs

    def field(offset, dtype, shape=(), strides=()):
        return np.ndarray((E,) + shape, dtype, buffer=buf, offset=offset, strides=(stride,) + strides)

    fs = (FRAME_SHAPE[1] * FRAME_SHAPE[2], FRAME_SHAPE[2], 1)
    stride = A3C_REPORT_BYTES
    v = dict(frame=field(A3C_REPORT_FRAME, np.uint8, FRAME_SHAPE, fs),
             next_state=field(A3C_REPORT_NEXT_STATE, np.uint8, FRAME_SHAPE, fs),
             uniform=field(A3C_REPORT_UNIFORM, np.float64), reward=field(A3C_REPORT_REWARD, np.float32),
             done=field(A3C_REPORT_DONE, np.uint8), reset=field(A3C_REPORT_RESET, np.uint8))
    stride = A3C_REPLY_BYTES
    base = E * A3C_REPORT_BYTES
    v.update(action=field(base + A3C_REPLY_ACTION, np.int32), max_prob=field(base + A3C_REPLY_MAX_PROB, np.float32))
    return v


# the Ape-X server's records (include/drl_b200.h: DRL_APEX_SERVER_*): two frames and a sample order per report
APEX_REPORT_FRAME, APEX_REPORT_NEXT_STATE, APEX_REPORT_EXPLORE, APEX_REPORT_REWARD, APEX_REPORT_DONE = (
    0, 28224, 56448, 56464, 56480)
APEX_REPORT_RESET, APEX_REPORT_ORDER, APEX_REPORT_BYTES = 56496, 56512, 58560
APEX_MAX_T = 512   # entries of the order field
APEX_REPLY_ACTION, APEX_REPLY_Q_ACTION, APEX_REPLY_BYTES = 0, 16, 32


def apex_exchange_bytes(num_envs):
    """Size of the Ape-X exchange block of num_envs environments: the reports, then the replies, rounded up to a
    page."""
    n = num_envs * (APEX_REPORT_BYTES + APEX_REPLY_BYTES)
    return -(-n // PAGE) * PAGE


def apex_exchange_views(buf, num_envs):
    """numpy views of the Ape-X records in the exchange block `buf` (a writable buffer of apex_exchange_bytes(num_envs)):
    frame, next_state, explore, reward, done, reset, order ([num_envs, 512]; the first T entries are read), action and
    q_action."""
    E = num_envs

    def field(offset, dtype, shape=(), strides=()):
        return np.ndarray((E,) + shape, dtype, buffer=buf, offset=offset, strides=(stride,) + strides)

    fs = (FRAME_SHAPE[1] * FRAME_SHAPE[2], FRAME_SHAPE[2], 1)
    stride = APEX_REPORT_BYTES
    v = dict(frame=field(APEX_REPORT_FRAME, np.uint8, FRAME_SHAPE, fs),
             next_state=field(APEX_REPORT_NEXT_STATE, np.uint8, FRAME_SHAPE, fs),
             explore=field(APEX_REPORT_EXPLORE, np.int32), reward=field(APEX_REPORT_REWARD, np.float32),
             done=field(APEX_REPORT_DONE, np.uint8), reset=field(APEX_REPORT_RESET, np.uint8),
             order=field(APEX_REPORT_ORDER, np.int32, (APEX_MAX_T,), (4,)))
    stride = APEX_REPLY_BYTES
    base = E * APEX_REPORT_BYTES
    v.update(action=field(base + APEX_REPLY_ACTION, np.int32), q_action=field(base + APEX_REPLY_Q_ACTION, np.float32))
    return v


def explore_action(rng, epsilon, num_action):
    """The epsilon-greedy draw of policy_handle.explore_actions for one environment, from its own RandomState `rng`:
    ``rng.rand() > epsilon`` keeps the greedy action (-1), otherwise ``rng.choice(num_action)`` is the action."""
    if rng.rand() > epsilon:
        return -1
    return int(rng.choice(num_action))


class _Stats:
    """The per-environment episode bookkeeping utils.impala_env_step updates."""

    def __init__(self, k):
        self.lives = [utils.START_LIVES] * k
        self.episode = [0] * k
        self.score = [0.0] * k
        self.episode_step = [0] * k
        self.total_max_prob = [0.0] * k


class _ApexStats:
    """The per-environment episode bookkeeping utils.apex_env_step updates."""

    def __init__(self, k):
        self.lives = [utils.START_LIVES] * k
        self.episode = [0] * k
        self.epsilon = [1.0] * k
        self.score = [0.0] * k
        self.episode_step = [0] * k
        self.total_max_prob = [0.0] * k


class _R2D2Stats:
    """The per-environment episode bookkeeping utils.r2d2_env_step updates."""

    def __init__(self, k):
        self.lives = [utils.START_LIVES] * k
        self.episode = [0] * k
        self.epsilon = [1.0] * k
        self.score = [0.0] * k
        self.episode_step = [0] * k
        self.episode_q_value = [0.0] * k


def _worker_loop(conn, shm, v, env_ids, env_fns, first_report, step):
    """The loop of every worker process: build the environments, write each one's first report (first_report(j, e,
    env)), signal ready, then per "go" step each environment (step(j, e, env) -> a finished episode or None) and signal
    ready with the finished episodes.  A failure is sent as ("error", task, traceback)."""
    task = env_ids[0]
    try:
        envs = []
        for j, fn in enumerate(env_fns):
            task = env_ids[j]
            envs.append(fn())
        start = first_report(envs)
        for j, e in enumerate(env_ids):
            task = e
            start(j, e, envs[j])
        info = dict(torch="torch" in sys.modules,
                    native="distributed_reinforcement_learning_b200._native" in sys.modules)
        conn.send(("ready", [], info))
        while conn.recv() == "go":
            finished = []
            for j, e in enumerate(env_ids):
                task = e
                episode = step(j, e, envs[j])
                if episode is not None:
                    finished.append(episode)
            conn.send(("ready", finished, None))
    except BaseException:
        try:
            conn.send(("error", task, traceback.format_exc()))
        except Exception:
            pass
    finally:
        del v
        shm.close()
        conn.close()


def _worker_main(conn, shm_name, num_envs, env_ids, env_fns, available_action, seeds, a3c=False):
    """An IMPALA worker process: k environments, each task env_ids[j] with its own RandomState(seeds[j]) for the uniform
    draws of its actions.  With `a3c` the records are the A3C server's, and after an episode end the worker also
    writes env.step's frame into next_state."""
    shm = shared_memory.SharedMemory(name=shm_name)
    v = (a3c_exchange_views if a3c else exchange_views)(shm.buf, num_envs)
    rngs, stats = [], None

    def first_report(envs):
        nonlocal stats
        rngs.extend(np.random.RandomState(s) for s in seeds)
        stats = _Stats(len(envs))

        def start(j, e, env):
            v["frame"][e] = env.reset()
            v["uniform"][e] = rngs[j].random_sample()
            v["reward"][e], v["done"][e], v["reset"][e] = 0.0, 0, 1
        return start

    def step(j, e, env):
        next_state, r, d, state, episode = utils.impala_env_step(env, int(v["action"][e]), available_action[j], stats,
                                                                 j, v["max_prob"][e], task=e)
        if a3c and episode is not None:
            v["next_state"][e] = next_state
        v["frame"][e] = state
        v["reward"][e], v["done"][e], v["reset"][e] = r, d, episode is not None
        v["uniform"][e] = rngs[j].random_sample()
        return episode

    _worker_loop(conn, shm, v, env_ids, env_fns, first_report, step)


def _a3c_worker_main(conn, shm_name, num_envs, env_ids, env_fns, available_action, seeds):
    """An A3C worker process: the IMPALA worker on the A3C records."""
    _worker_main(conn, shm_name, num_envs, env_ids, env_fns, available_action, seeds, a3c=True)


def _r2d2_worker_main(conn, shm_name, num_envs, env_ids, env_fns, num_action, channels, seeds):
    """An R2D2 worker process: k environments, each task env_ids[j] with its own RandomState(seeds[j]) for its explore
    decisions and random actions (explore_action)."""
    shm = shared_memory.SharedMemory(name=shm_name)
    v = r2d2_exchange_views(shm.buf, num_envs, channels)
    rngs, stats = [], None

    def first_report(envs):
        nonlocal stats
        rngs.extend(np.random.RandomState(s) for s in seeds)
        stats = _R2D2Stats(len(envs))

        def start(j, e, env):
            v["frame"][e] = env.reset()
            v["explore"][e] = explore_action(rngs[j], stats.epsilon[j], num_action)
            v["reward"][e], v["done"][e], v["reset"][e] = 0.0, 0, 1
        return start

    def step(j, e, env):
        _, r, d, state, episode = utils.r2d2_env_step(env, int(v["action"][e]), stats, j, v["q_action"][e], task=e)
        v["frame"][e] = state
        v["reward"][e], v["done"][e], v["reset"][e] = r, d, episode is not None
        v["explore"][e] = explore_action(rngs[j], stats.epsilon[j], num_action)
        return episode

    _worker_loop(conn, shm, v, env_ids, env_fns, first_report, step)


def _apex_worker_main(conn, shm_name, num_envs, env_ids, env_fns, available_action, num_action, trajectory,
                      buffer_capacity, seeds):
    """An Ape-X worker process: k environments, each task env_ids[j] with its own RandomState(seeds[j]) and a count of
    its LocalBuffer's length.  Per step, in the reference actor's order: env.step, then (once the buffer holds more
    than 3 T transitions) the sample order's permutation draw, then the explore draw of the next act
    (explore_action)."""
    shm = shared_memory.SharedMemory(name=shm_name)
    v = apex_exchange_views(shm.buf, num_envs)
    T = int(trajectory)
    rngs, stats, length = [], None, []

    def first_report(envs):
        nonlocal stats
        rngs.extend(np.random.RandomState(s) for s in seeds)
        stats = _ApexStats(len(envs))
        length.extend([0] * len(envs))

        def start(j, e, env):
            v["frame"][e] = env.reset()
            v["explore"][e] = explore_action(rngs[j], stats.epsilon[j], num_action)
            v["reward"][e], v["done"][e], v["reset"][e] = 0.0, 0, 1
        return start

    def step(j, e, env):
        next_state, r, d, state, episode = utils.apex_env_step(env, int(v["action"][e]), available_action[j], stats,
                                                               j, v["q_action"][e], task=e)
        length[j] = min(length[j] + 1, buffer_capacity)
        if length[j] > 3 * T:   # LocalBuffer.sample's draw
            v["order"][e, :T] = rngs[j].permutation(length[j])[:T]
        if episode is not None:
            v["next_state"][e] = next_state
        v["frame"][e] = state
        v["reward"][e], v["done"][e], v["reset"][e] = r, d, episode is not None
        v["explore"][e] = explore_action(rngs[j], stats.epsilon[j], num_action)
        return episode

    _worker_loop(conn, shm, v, env_ids, env_fns, first_report, step)


class EnvWorkerPool:
    """``len(env_fns)`` environments (1..256) in spawned worker processes of ``envs_per_worker`` environments each.

    Environment i is task i: ``env_fns[i]()`` builds it in its worker, it steps under ``utils.impala_env_step`` with
    ``available_action[i]``, and the uniform draws of its actions come from ``np.random.RandomState(seeds[i])``, so
    they do not depend on batching or on how environments are grouped into workers.  The env factories must be
    picklable (ValueError otherwise).  The workers import neither torch nor CUDA.

    ``close()`` (also on leaving a ``with`` block) first closes every ``PolicyServer`` still bound to the pool (each
    has the exchange block registered with CUDA), then stops every worker, terminating the ones that do not exit in
    time, and frees the exchange block."""

    def __init__(self, env_fns, available_action, envs_per_worker, seeds, start_timeout=300.0, join_timeout=10.0):
        env_fns, seeds = list(env_fns), [int(s) for s in seeds]
        available_action = [int(a) for a in available_action]
        self._check(env_fns, envs_per_worker)
        if len(available_action) != len(env_fns) or len(seeds) != len(env_fns):
            raise ValueError("available_action and seeds need one entry per environment (%d)" % len(env_fns))
        self._start(env_fns, envs_per_worker, seeds, exchange_bytes, exchange_views, _worker_main,
                    lambda lo, hi: (available_action[lo:hi],), start_timeout, join_timeout)

    @staticmethod
    def _check(env_fns, envs_per_worker):
        n = len(env_fns)
        if not 1 <= n <= MAX_ENVS:
            raise ValueError("%d environments, a pool serves 1..%d" % (n, MAX_ENVS))

    def _start(self, env_fns, envs_per_worker, seeds, size, views, target, worker_args, start_timeout, join_timeout):
        """Checks envs_per_worker and the factories, makes the exchange block (size(n): its bytes; views(buf, n): its
        numpy views) and spawns one `target` process per envs_per_worker environments, with the arguments (pipe, block
        name, n, env ids, env factories, *worker_args(lo, hi), seeds) of environments lo..hi-1; waits for every
        worker's first report."""
        n, k = len(env_fns), int(envs_per_worker)
        if k < 1:
            raise ValueError("envs_per_worker must be >= 1 (got %d)" % k)
        for i, fn in enumerate(env_fns):
            try:
                pickle.dumps(fn)
            except Exception as e:
                raise ValueError("env_fns[%d] cannot be pickled for a spawned worker: %s" % (i, e)) from None
        self.num_envs, self.envs_per_worker = n, k
        self.join_timeout = join_timeout
        self.exchange_bytes = size(n)
        self._workers = []
        self._pending = set()
        self._servers = []
        self._shm = shared_memory.SharedMemory(create=True, size=self.exchange_bytes)
        self.views = views(self._shm.buf, n)
        self._anchor = C.c_char.from_buffer(self._shm.buf)
        self.address = C.addressof(self._anchor)
        self.worker_info = []
        try:
            ctx = mp.get_context("spawn")
            for w in range(0, n, k):
                ids = list(range(w, min(n, w + k)))
                parent, child = ctx.Pipe()
                p = ctx.Process(target=target, name="env-worker-%d" % (w // k),
                                args=(child, self._shm.name, n, ids, env_fns[w:w + k], *worker_args(w, w + k),
                                      seeds[w:w + k]), daemon=True)
                p.start()
                child.close()
                self._workers.append(dict(process=p, conn=parent, env_ids=ids))
            while len(self.worker_info) < len(self._workers):
                if not self._collect(start_timeout):
                    raise RuntimeError("environment workers did not start within %.0f s" % start_timeout)
        except BaseException:
            self.close()
            raise

    @property
    def num_workers(self):
        return len(self._workers)

    def env_ids(self, w):
        return self._workers[w]["env_ids"]

    def _collect(self, timeout, finished=None):
        """Receives the reports of the workers that have one ready, waiting up to `timeout` s (None: forever) for the
        first; -> whether any arrived."""
        waiting = {id(x["conn"]): w for w, x in enumerate(self._workers) if w not in self._pending}
        conns = [self._workers[w]["conn"] for w in waiting.values()]
        ready = mp.connection.wait(conns, timeout) if conns else []
        for c in ready:
            w = waiting[id(c)]
            ids = self._workers[w]["env_ids"]
            try:
                kind, a, b = c.recv()
            except (EOFError, OSError):
                raise RuntimeError("environment worker %d (tasks %s) exited without a report (exit code %s)"
                                   % (w, ids, self._workers[w]["process"].exitcode)) from None
            if kind == "error":
                raise RuntimeError("environment task %d raised in worker %d:\n%s" % (a, w, b))
            if b is not None:
                self.worker_info.append(b)
            if finished is not None:
                finished.extend(a)
            self._pending.add(w)
        return bool(ready)

    def wait_ready(self, timeout=None):
        """Waits up to `timeout` s (None: forever) until at least one worker has reported, and takes every report
        that is ready.  -> (the workers whose reports await a reply, in worker order; the episodes they finished)."""
        finished = []
        if not self._pending:
            self._collect(timeout, finished)
        self._collect(0, finished)
        return sorted(self._pending), finished

    def reply(self, workers):
        """Tells these workers that their reply records are written."""
        for w in workers:
            self._pending.discard(w)
            self._workers[w]["conn"].send("go")

    def _bind(self, server):
        """Called by a PolicyServer that registered the exchange block: close() closes it before freeing the block."""
        if getattr(self, "_shm", None) is None:
            raise ValueError("the pool is closed")
        self._servers.append(server)

    def _unbind(self, server):
        self._servers = [s for s in self._servers if s is not server]

    def close(self):
        for server in list(getattr(self, "_servers", ())):
            server.close()
        for x in self._workers:
            try:
                x["conn"].send("stop")
            except Exception:
                pass
        for x in self._workers:
            p = x["process"]
            p.join(self.join_timeout)
            if p.is_alive():
                p.terminate()
                p.join(self.join_timeout)
            if p.is_alive():
                p.kill()
                p.join()
            x["conn"].close()
        self._workers, self._pending = [], set()
        if getattr(self, "_shm", None) is not None:
            self.views = None
            self._anchor = None
            self._shm.close()
            self._shm.unlink()
            self._shm = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class R2D2EnvWorkerPool(EnvWorkerPool):
    """``len(env_fns)`` R2D2 environments (1..256) in spawned worker processes of ``envs_per_worker`` environments
    each, for an ``R2D2PolicyServer``.

    Environment i is task i: ``env_fns[i]()`` builds it in its worker (its frames are 84x84x``channels``), it steps
    under ``utils.r2d2_env_step`` with the raw action, and its explore decisions and random actions in [0,
    ``num_action``) come from ``np.random.RandomState(seeds[i])`` by the rule of ``policy_handle.explore_actions``
    (``explore_action``), so they do not depend on batching or on how environments are grouped into workers.  The
    reports and replies are the R2D2 records (``r2d2_exchange_views``); everything else -- the pipes, ``wait_ready``,
    ``reply``, the failure reports and ``close()`` -- is ``EnvWorkerPool``'s."""

    def __init__(self, env_fns, num_action, envs_per_worker, seeds, channels=1, start_timeout=300.0,
                 join_timeout=10.0):
        env_fns, seeds = list(env_fns), [int(s) for s in seeds]
        num_action, channels = int(num_action), int(channels)
        self._check(env_fns, envs_per_worker)
        if len(seeds) != len(env_fns):
            raise ValueError("seeds need one entry per environment (%d)" % len(env_fns))
        if num_action < 2:
            raise ValueError("num_action must be >= 2 (got %d)" % num_action)
        if channels not in (1, 4):
            raise ValueError("channels must be 1 or 4 (got %d)" % channels)
        self.num_action, self.channels = num_action, channels
        self._start(env_fns, envs_per_worker, seeds, exchange_bytes,
                    lambda buf, n: r2d2_exchange_views(buf, n, channels), _r2d2_worker_main,
                    lambda lo, hi: (num_action, channels), start_timeout, join_timeout)


class A3CEnvWorkerPool(EnvWorkerPool):
    """``len(env_fns)`` A3C environments (1..256) in spawned worker processes of ``envs_per_worker`` environments each,
    for an ``A3CPolicyServer``.

    Environment i is task i: ``env_fns[i]()`` builds it in its worker, it steps under ``utils.impala_env_step`` with
    ``available_action[i]`` -- the IMPALA rule is exactly the A3C actor's (train_a3c.py:150-178: the step with
    ``action % available_action``, a lost life stored as reward -1 and done, the counters and the previous action reset
    at an episode's end) -- and the uniform draws of its actions come from ``np.random.RandomState(seeds[i])``, drawn as
    the IMPALA worker draws them, so they do not depend on batching or on how environments are grouped into workers.
    The reports and replies are the A3C records (``a3c_exchange_views``); after an episode end the worker also writes
    env.step's frame into next_state.  Everything else -- the pipes, ``wait_ready``, ``reply``, the failure reports and
    ``close()`` -- is ``EnvWorkerPool``'s."""

    def __init__(self, env_fns, available_action, envs_per_worker, seeds, start_timeout=300.0, join_timeout=10.0):
        env_fns, seeds = list(env_fns), [int(s) for s in seeds]
        available_action = [int(a) for a in available_action]
        self._check(env_fns, envs_per_worker)
        if len(available_action) != len(env_fns) or len(seeds) != len(env_fns):
            raise ValueError("available_action and seeds need one entry per environment (%d)" % len(env_fns))
        self._start(env_fns, envs_per_worker, seeds, a3c_exchange_bytes, a3c_exchange_views, _a3c_worker_main,
                    lambda lo, hi: (available_action[lo:hi],), start_timeout, join_timeout)


class ApexEnvWorkerPool(EnvWorkerPool):
    """``len(env_fns)`` Ape-X environments (1..256) in spawned worker processes of ``envs_per_worker`` environments
    each, for an ``ApexPolicyServer``.

    Environment i is task i: ``env_fns[i]()`` builds it in its worker, it steps under ``utils.apex_env_step`` with
    ``available_action[i]``, and every draw of its actor -- the explore decision and random action in [0,
    ``num_action``) of each act (``explore_action``), and the sample order of each push (``LocalBuffer.sample``'s
    ``permutation``, once its ``LocalBuffer(buffer_capacity)`` holds more than 3 ``trajectory`` transitions) -- comes
    from ``np.random.RandomState(seeds[i])`` in the reference actor's order, so the draws do not depend on batching or
    on how environments are grouped into workers.  The buffers themselves live on the GPU, in the server; a worker
    counts its length.  The reports and replies are the Ape-X records (``apex_exchange_views``); after an episode end
    the worker also writes env.step's frame into next_state.  Everything else -- the pipes, ``wait_ready``, ``reply``,
    the failure reports and ``close()`` -- is ``EnvWorkerPool``'s."""

    def __init__(self, env_fns, available_action, num_action, envs_per_worker, seeds, trajectory,
                 buffer_capacity=int(1e4), start_timeout=300.0, join_timeout=10.0):
        env_fns, seeds = list(env_fns), [int(s) for s in seeds]
        available_action = [int(a) for a in available_action]
        num_action, trajectory, buffer_capacity = int(num_action), int(trajectory), int(buffer_capacity)
        self._check(env_fns, envs_per_worker)
        if len(available_action) != len(env_fns) or len(seeds) != len(env_fns):
            raise ValueError("available_action and seeds need one entry per environment (%d)" % len(env_fns))
        if num_action < 2:
            raise ValueError("num_action must be >= 2 (got %d)" % num_action)
        if not 1 <= trajectory <= APEX_MAX_T:
            raise ValueError("trajectory must be in [1, %d] (got %d)" % (APEX_MAX_T, trajectory))
        if buffer_capacity <= 3 * trajectory:
            raise ValueError("buffer_capacity %d must exceed 3 trajectory = %d (a buffer pushes once it holds more "
                             "than 3 trajectory transitions)" % (buffer_capacity, 3 * trajectory))
        self.num_action, self.trajectory, self.buffer_capacity = num_action, trajectory, buffer_capacity
        self._start(env_fns, envs_per_worker, seeds, apex_exchange_bytes, apex_exchange_views, _apex_worker_main,
                    lambda lo, hi: (available_action[lo:hi], num_action, trajectory, buffer_capacity),
                    start_timeout, join_timeout)


class _ServerBase:
    """What PolicyServer, R2D2PolicyServer, A3CPolicyServer and ApexPolicyServer share: the binding to a pool, the
    serve lock, the C handle's lifetime, the policy sync before a serve, and the serve loop.  A family sets `_prefix`
    (its ``drl_<prefix>_*`` entry points) and `_what` (its name in messages) and implements ``_learner_step``; the
    create call takes (policy, queue, num_envs, *create_args, block, block size, out)."""
    _prefix = None
    _what = None

    def _bind_and_create(self, policy, queue, pool, learner, *create_args):
        from . import _native as N
        from . import dp
        if dp.distributed():
            raise RuntimeError("%s is single-replica: the queue lives on one device" % type(self).__name__)
        self._N = N
        self.policy, self.queue, self.pool, self.learner = policy, queue, pool, learner
        self.batch_sizes = collections.Counter()
        self.syncs = 0
        self._synced_step = None
        self._todo, self._workers, self._finished = [], [], []
        self._lock = threading.Lock()   # a serve and close() never overlap
        self._s = C.c_void_p()
        bind = getattr(pool, "_bind", None)
        if bind is not None:
            bind(self)
        try:
            N.check(self._fn("create")(policy._h, queue._q, pool.num_envs, *create_args, C.c_void_p(pool.address),
                                       pool.exchange_bytes, C.byref(self._s)))
        except BaseException:
            self.close()
            raise

    def _fn(self, name):
        return getattr(self._N.lib, "drl_%s_%s" % (self._prefix, name))

    def close(self):
        """Destroys the server (unregistering the exchange block); waits for a serve in progress."""
        with self._lock:
            if self._s.value:
                self._fn("destroy")(self._s)
                self._s = C.c_void_p()
        unbind = getattr(getattr(self, "pool", None), "_unbind", None)
        if unbind is not None:
            unbind(self)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _learner_step(self):
        raise NotImplementedError

    def _sync(self):
        if self.learner is None:
            return
        step = self._learner_step()
        if step != self._synced_step:
            self.learner.sync_policy(self.policy)
            self._synced_step = step
            self.syncs += 1

    def serve(self, env_ids, timeout_ms=-1):
        """One ``drl_<prefix>_serve`` of these environments (at most max_batch, distinct)."""
        ids = np.ascontiguousarray(env_ids, np.int32)
        N = self._N
        with self._lock:
            if not self._s.value:
                raise ValueError("the %s is closed" % self._what)
            N.check(self._fn("serve")(self._s, int(ids.size), N.ptr(ids), int(timeout_ms)))
        self.batch_sizes[int(ids.size)] += 1

    def serve_once(self, wait=None, timeout_ms=-1):
        """Serves every report that is ready, waiting up to `wait` s (None: forever) for the first.  A serve blocked
        by a full queue for `timeout_ms` (>= 0) raises ``TimeoutError_``; the reports not yet served then wait for the
        next call.  -> the episodes that finished."""
        if not self._todo:
            self._workers, finished = self.pool.wait_ready(wait)
            self._finished += finished
            self._todo = [e for w in self._workers for e in self.pool.env_ids(w)]
        if self._todo:
            self._sync()
        mb = self.policy.max_batch
        while self._todo:
            self.serve(self._todo[:mb], timeout_ms)
            self._todo = self._todo[mb:]
        self.pool.reply(self._workers)
        self._workers = []
        out, self._finished = self._finished, []
        return out

    def run(self, stop, on_episodes=None):
        """serve_once until the threading.Event `stop` is set; `on_episodes` (if given) receives each non-empty list
        of finished episodes."""
        N = self._N
        while not stop.is_set():
            try:
                episodes = self.serve_once(wait=0.05, timeout_ms=100)
            except N.TimeoutError_:
                continue
            if episodes and on_episodes is not None:
                on_episodes(episodes)


class PolicyServer(_ServerBase):
    """Serves the environments of an ``EnvWorkerPool`` from one ``NativePolicy`` into one ``DeviceFIFOQueue``.

    ``serve_once`` waits for at least one worker's reports, takes every report that is ready and serves them in
    chunks of ``policy.max_batch`` environments (no batching knob: batches grow with load), then answers the workers.
    Before a serve it syncs the policy from ``learner`` (an ``impala.Agent``) whenever the learner has trained since
    the last sync, so parameters can change inside an unroll; each trajectory records the policy that acted, which is
    what V-trace corrects for.  While the queue is full a serve blocks: that is the workers' backpressure.
    ``batch_sizes`` counts the served batches by size.  Single-replica, like ``train_from_queue``.  Closing the pool
    closes its server first, so the exchange block is never freed while CUDA has it registered.  ``serve_once``
    returns the finished episodes as dicts of task, episode, score, episode_step and prob (the values
    train_impala.py:170-172 logs)."""
    _prefix = "policy_server"
    _what = "policy server"

    def __init__(self, policy, queue, pool, learner=None):
        from .distributed_queue.buffer_queue import DeviceFIFOQueue
        if not isinstance(queue, DeviceFIFOQueue):
            raise TypeError("PolicyServer: queue must be a DeviceFIFOQueue, got %s" % type(queue).__name__)
        self._bind_and_create(policy, queue, pool, learner)

    def _learner_step(self):
        return self.learner.num_env_frames


class R2D2PolicyServer(_ServerBase):
    """Serves the environments of an ``R2D2EnvWorkerPool`` from one ``NativeR2D2Policy`` into one
    ``R2D2DeviceFIFOQueue``, which ``r2d2.DeviceMemory.add_from_queue`` ingests.

    ``serve``, ``serve_once``, ``run`` and ``close`` are ``PolicyServer``'s; the explore decisions come with the
    reports.  Before a serve it syncs the policy from ``learner`` (an ``r2d2.Agent``) whenever the learner has trained
    (``train_calls``) since the last sync.  The reference's actor runs ``parameter_sync`` once per sequence; here the
    sync follows the learner, so one sequence may be recorded under several parameter versions.  R2D2 learns
    off-policy from replay, and the stored (h, c) of a sequence's step 0 is burnt in again by the learner, so this
    changes which parameters acted, not what the learner computes from a sequence.  While the queue is full a serve
    blocks.  Single-replica, like the device replay memory.  Closing the pool closes its server first.  ``serve_once``
    returns the finished episodes as dicts of task, episode, score, epsilon, episode_step and avg_q_value (the values
    train_r2d2.py:227-230 logs)."""
    _prefix = "r2d2_policy_server"
    _what = "r2d2 policy server"

    def __init__(self, policy, queue, pool, learner=None):
        from .distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
        from .r2d2_policy import NativeR2D2Policy
        if not isinstance(policy, NativeR2D2Policy):
            raise TypeError("R2D2PolicyServer: policy must be a NativeR2D2Policy, got %s" % type(policy).__name__)
        if not isinstance(queue, R2D2DeviceFIFOQueue):
            raise TypeError("R2D2PolicyServer: queue must be an R2D2DeviceFIFOQueue, got %s" % type(queue).__name__)
        channels = getattr(pool, "channels", None)
        if channels is not None and channels != queue.input_shape[2]:
            raise ValueError("R2D2PolicyServer: the pool's environments give 84x84x%d frames, the queue stores 84x84x%d"
                             % (channels, queue.input_shape[2]))
        if learner is not None and getattr(learner, "lstm_size", policy.L) != policy.L:
            raise ValueError("R2D2PolicyServer: the learner has lstm_size %d, the policy %d: the policy engine syncs "
                             "from a learner of its own width" % (learner.lstm_size, policy.L))
        self._bind_and_create(policy, queue, pool, learner)

    def _learner_step(self):
        return self.learner.train_calls


class A3CPolicyServer(_ServerBase):
    """Serves the environments of an ``A3CEnvWorkerPool`` from one ``NativeA3CPolicy`` into one
    ``A3CDeviceFIFOQueue``, which ``a3c.Agent.train_from_queue`` trains from.

    ``serve``, ``serve_once``, ``run`` and ``close`` are ``PolicyServer``'s; the uniform draws come with the reports.
    Before a serve it syncs the policy from ``learner`` (an ``a3c.Agent``) whenever the learner has trained
    (``num_env_frames``, its step counter) since the last sync.  The reference's actor runs ``parameter_sync`` once per
    unroll, so each of its trajectories is recorded under one parameter version; here the sync follows the learner, so
    one unroll may be recorded under several versions.  A3C has no off-policy correction; the lag is bounded by how far
    acting runs ahead of training, which the queue's capacity limits as the reference's queue does.  While the queue is
    full a serve blocks.  Single-replica, like ``train_from_queue``.  Closing the pool closes its server first.
    ``serve_once`` returns the finished episodes as dicts of task, episode, prob, score and episode_step (the keys
    ``A3CVectorActor.run_unroll`` returns)."""
    _prefix = "a3c_policy_server"
    _what = "a3c policy server"

    def __init__(self, policy, queue, pool, learner=None):
        from .apex_policy import NativeA3CPolicy
        from .distributed_queue.buffer_queue import A3CDeviceFIFOQueue
        if not isinstance(policy, NativeA3CPolicy):
            raise TypeError("A3CPolicyServer: policy must be a NativeA3CPolicy, got %s" % type(policy).__name__)
        if not isinstance(queue, A3CDeviceFIFOQueue):
            raise TypeError("A3CPolicyServer: queue must be an A3CDeviceFIFOQueue, got %s" % type(queue).__name__)
        self._bind_and_create(policy, queue, pool, learner)

    def _learner_step(self):
        return self.learner.num_env_frames


class ApexPolicyServer(_ServerBase):
    """Serves the environments of an ``ApexEnvWorkerPool`` from one ``NativeApexPolicy`` into one
    ``ApexDeviceFIFOQueue``, which ``apex.DeviceMemory.add_from_queue`` ingests.

    Each environment's ``LocalBuffer(pool.buffer_capacity)`` is a ring on the GPU (565 MB per environment at capacity
    1e4): a serve completes each environment's previous transition there and, once its buffer holds more than 3 T
    transitions, pushes the sample the worker drew as one queue record, on the device.  ``serve``, ``serve_once``,
    ``run`` and ``close`` are ``PolicyServer``'s; the explore actions and sample orders come with the reports.  Before
    a serve it syncs the policy from ``learner`` (an ``apex.Agent``) whenever the learner has trained
    (``num_env_frames``) since the last sync.  The reference's actor runs ``parameter_sync`` once per unroll of T steps;
    here the sync follows the learner.  Ape-X learns off-policy from replay, so this changes which parameters acted,
    not what the learner computes from a transition.  While the queue is full a serve blocks.  Single-replica, like the
    device replay memory.  Closing the pool closes its server first.  ``serve_once`` returns the finished episodes as
    dicts of task, episode, score, epsilon, episode_step and total_max_prob (the values train_apex.py:215-220 logs).
    ``read(env, j)`` copies deque index j of an environment's buffer, for tests."""
    _prefix = "apex_policy_server"
    _what = "apex policy server"

    def __init__(self, policy, queue, pool, learner=None):
        from .apex_policy import NativeApexPolicy
        from .distributed_queue.buffer_queue import ApexDeviceFIFOQueue
        if not isinstance(policy, NativeApexPolicy):
            raise TypeError("ApexPolicyServer: policy must be a NativeApexPolicy, got %s" % type(policy).__name__)
        if not isinstance(queue, ApexDeviceFIFOQueue):
            raise TypeError("ApexPolicyServer: queue must be an ApexDeviceFIFOQueue, got %s" % type(queue).__name__)
        T = getattr(pool, "trajectory", None)
        if T is not None and T != queue.trajectory:
            raise ValueError("ApexPolicyServer: the pool's workers sample %d transitions, the queue records %d"
                             % (T, queue.trajectory))
        self.capacity = int(pool.buffer_capacity)
        self._bind_and_create(policy, queue, pool, learner, self.capacity)

    def _learner_step(self):
        return self.learner.num_env_frames

    def read(self, env, j):
        """Deque index j of environment env's buffer as a dict of state, next_state, previous_action, action, reward,
        done."""
        N = self._N
        out = dict(state=np.empty(FRAME_SHAPE, np.uint8), next_state=np.empty(FRAME_SHAPE, np.uint8),
                   previous_action=np.empty(1, np.int32), action=np.empty(1, np.int32),
                   reward=np.empty(1, np.float32), done=np.empty(1, np.uint8))
        with self._lock:
            if not self._s.value:
                raise ValueError("the %s is closed" % self._what)
            N.check(self._fn("read")(self._s, int(env), int(j), *[N.ptr(a) for a in out.values()]))
        return dict(state=out["state"], next_state=out["next_state"], previous_action=int(out["previous_action"][0]),
                    action=int(out["action"][0]), reward=float(out["reward"][0]), done=bool(out["done"][0]))
