"""One tiny learner step per math mode for compute-sanitizer (memcheck / racecheck / synccheck of the mbarrier + wgmma
pipelines), with --peer under torchrun the 2-GPU fused exchange (flag protocol over NVLink peer memory), and with
--serve one eager serve loop of the IMPALA policy server (drl_policy_server_*: gather, per-row commit, act, scatter)
over a registered exchange block the script fills itself, without worker processes, and with --serve-r2d2 and
--serve-a3c the same for the R2D2 policy server (drl_r2d2_policy_server_*) and the A3C policy server
(drl_a3c_policy_server_*).

    compute-sanitizer --tool memcheck  python tools/sanitize_step.py --modes 2 3
    compute-sanitizer --tool racecheck python tools/sanitize_step.py --modes 2
    torchrun --nproc-per-node 2 ... tools/sanitize_step.py --peer      (run each rank under compute-sanitizer)
    DRL_B200_CUDA_GRAPH=0 compute-sanitizer --tool memcheck python tools/sanitize_step.py --serve
    DRL_B200_CUDA_GRAPH=0 compute-sanitizer --tool memcheck python tools/sanitize_step.py --serve-r2d2
    DRL_B200_CUDA_GRAPH=0 compute-sanitizer --tool memcheck python tools/sanitize_step.py --serve-a3c
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def serve_loop(envs=6, max_batch=4, trajectory=3, unrolls=3):
    """Serves `envs` environments for `unrolls` unrolls in random subsets of at most max_batch, with reset flags now
    and then, and checks the committed trajectories' frames against the reports."""
    import ctypes as C
    import mmap
    from distributed_reinforcement_learning_b200.actor_server import PolicyServer, exchange_bytes, exchange_views
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.model import impala_actor_critic as model
    from distributed_reinforcement_learning_b200.policy import NativePolicy

    class Block:   # the exchange block of a pool, without workers
        def __init__(self):
            self.num_envs, self.exchange_bytes = envs, exchange_bytes(envs)
            self.mem = mmap.mmap(-1, self.exchange_bytes)
            self.anchor = C.c_char.from_buffer(self.mem)
            self.address = C.addressof(self.anchor)
            self.views = exchange_views(self.mem, envs)

    graph = os.environ.get("DRL_B200_CUDA_GRAPH", "1") != "0"
    rng = np.random.RandomState(0)
    pol = NativePolicy(max_batch, num_action=18, use_cuda_graph=graph)
    pol.set_params(model.init_params(seed=0))
    q = DeviceFIFOQueue(trajectory, (84, 84, 4), 18, envs * unrolls, envs, 1, 256)
    blk = Block()
    v = blk.views
    server = PolicyServer(pol, q, blk)
    frames = {e: [] for e in range(envs)}
    for step in range(unrolls * trajectory + 1):
        for e in range(envs):
            v["frame"][e] = rng.randint(0, 256, (84, 84, 4))
            v["uniform"][e] = rng.random_sample()
            v["reward"][e], v["done"][e], v["reset"][e] = rng.randint(3), rng.rand() < 0.2, step == 0 or rng.rand() < 0.1
            frames[e].append(v["frame"][e].copy())
        ids = rng.permutation(envs).astype(np.int32)
        k = 0
        while k < envs:
            c = rng.randint(1, max_batch + 1)
            server.serve(ids[k:k + c])
            k += c
        assert ((v["action"][:envs] >= 0) & (v["action"][:envs] < 18)).all()
    assert q.get_size() == envs * unrolls
    want = {np.stack(frames[e][u * trajectory:(u + 1) * trajectory]).tobytes()
            for e in range(envs) for u in range(unrolls)}
    got = {q.read(j)["state"].tobytes() for j in range(envs * unrolls)}
    assert got == want
    server.close()
    q.close()
    pol.close()
    print("serve loop (cuda graph %s): %d serves of %d environments, %d trajectories committed ok"
          % (graph, unrolls * trajectory + 1, envs, envs * unrolls), flush=True)


def serve_r2d2_loop(envs=6, max_batch=4, seq_len=3, unrolls=3, channels=1, num_action=4):
    """Serves `envs` R2D2 environments for `unrolls` sequences in random subsets of at most max_batch, with explore
    actions and reset flags now and then, and checks the committed sequences' frames and actions against the reports
    and replies."""
    import ctypes as C
    import mmap
    from distributed_reinforcement_learning_b200.actor_server import (R2D2PolicyServer, exchange_bytes,
                                                                      r2d2_exchange_views)
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import R2D2DeviceFIFOQueue
    from distributed_reinforcement_learning_b200.model import r2d2_lstm as model
    from distributed_reinforcement_learning_b200.r2d2_policy import NativeR2D2Policy

    class Block:   # the exchange block of a pool, without workers
        def __init__(self):
            self.num_envs, self.exchange_bytes = envs, exchange_bytes(envs)
            self.mem = mmap.mmap(-1, self.exchange_bytes)
            self.anchor = C.c_char.from_buffer(self.mem)
            self.address = C.addressof(self.anchor)
            self.views = r2d2_exchange_views(self.mem, envs, channels)

    shape = (84, 84, channels)
    graph = os.environ.get("DRL_B200_CUDA_GRAPH", "1") != "0"
    rng = np.random.RandomState(0)
    pol = NativeR2D2Policy(max_batch, num_action=num_action, input_shape=shape, use_cuda_graph=graph)
    pol.set_params(model.init_params(0, num_action=num_action, lstm_size=64, input_shape=shape))
    q = R2D2DeviceFIFOQueue(seq_len, shape, num_action, envs * unrolls, envs, 1, 64)
    blk = Block()
    v = blk.views
    server = R2D2PolicyServer(pol, q, blk)
    frames = {e: [] for e in range(envs)}
    actions = {e: [] for e in range(envs)}
    for step in range(unrolls * seq_len + 1):
        for e in range(envs):
            v["frame"][e] = rng.randint(0, 256, shape)
            v["explore"][e] = rng.randint(0, num_action) if rng.rand() < 0.3 else -1
            v["reward"][e], v["done"][e], v["reset"][e] = rng.randint(3), rng.rand() < 0.2, step == 0 or rng.rand() < 0.1
            frames[e].append(v["frame"][e].copy())
        ids = rng.permutation(envs).astype(np.int32)
        k = 0
        while k < envs:
            c = rng.randint(1, max_batch + 1)
            server.serve(ids[k:k + c])
            k += c
        assert ((v["action"][:envs] >= 0) & (v["action"][:envs] < num_action)).all()
        explore = v["explore"][:envs]
        assert (v["action"][:envs][explore >= 0] == explore[explore >= 0]).all()
        for e in range(envs):
            actions[e].append(int(v["action"][e]))
    assert q.get_size() == envs * unrolls
    want = {(np.stack(frames[e][u * seq_len:(u + 1) * seq_len]).tobytes(),
             np.array(actions[e][u * seq_len:(u + 1) * seq_len], np.int32).tobytes())
            for e in range(envs) for u in range(unrolls)}
    got = {(r["state"].tobytes(), r["action"].tobytes()) for r in (q.read(j) for j in range(envs * unrolls))}
    assert got == want
    server.close()
    q.close()
    pol.close()
    print("r2d2 serve loop (cuda graph %s): %d serves of %d environments, %d sequences committed ok"
          % (graph, unrolls * seq_len + 1, envs, envs * unrolls), flush=True)


def serve_a3c_loop(envs=6, max_batch=4, trajectory=3, unrolls=3, num_action=4):
    """Serves `envs` A3C environments for `unrolls` unrolls in random subsets of at most max_batch, with reset flags
    (and next_state frames) now and then, and checks the committed unrolls' state and next_state frames and actions
    against the reports and replies."""
    import ctypes as C
    import mmap
    from distributed_reinforcement_learning_b200.actor_server import (A3CPolicyServer, a3c_exchange_bytes,
                                                                      a3c_exchange_views)
    from distributed_reinforcement_learning_b200.apex_policy import NativeA3CPolicy
    from distributed_reinforcement_learning_b200.distributed_queue.buffer_queue import A3CDeviceFIFOQueue
    from distributed_reinforcement_learning_b200.model import actor_critic as model

    class Block:   # the exchange block of a pool, without workers
        def __init__(self):
            self.num_envs, self.exchange_bytes = envs, a3c_exchange_bytes(envs)
            self.mem = mmap.mmap(-1, self.exchange_bytes)
            self.anchor = C.c_char.from_buffer(self.mem)
            self.address = C.addressof(self.anchor)
            self.views = a3c_exchange_views(self.mem, envs)

    shape = (84, 84, 4)
    graph = os.environ.get("DRL_B200_CUDA_GRAPH", "1") != "0"
    rng = np.random.RandomState(0)
    pol = NativeA3CPolicy(max_batch, num_action=num_action, input_shape=shape, use_cuda_graph=graph)
    pol.set_params(model.init_params(0, num_action=num_action, input_shape=shape))
    q = A3CDeviceFIFOQueue(trajectory, shape, num_action, envs, queue_size=envs * unrolls)
    blk = Block()
    v = blk.views
    server = A3CPolicyServer(pol, q, blk)
    frames = {e: [] for e in range(envs)}
    nexts = {e: [] for e in range(envs)}
    actions = {e: [] for e in range(envs)}
    for step in range(unrolls * trajectory + 1):
        for e in range(envs):
            v["frame"][e] = rng.randint(0, 256, shape)
            reset = step == 0 or rng.rand() < 0.2
            if reset and step > 0:
                v["next_state"][e] = rng.randint(0, 256, shape)
            v["uniform"][e] = rng.random_sample()
            v["reward"][e], v["done"][e], v["reset"][e] = rng.randint(3), rng.rand() < 0.2, reset
            if step > 0:
                nexts[e].append((v["next_state"][e] if reset else v["frame"][e]).copy())
            frames[e].append(v["frame"][e].copy())
        ids = rng.permutation(envs).astype(np.int32)
        k = 0
        while k < envs:
            c = rng.randint(1, max_batch + 1)
            server.serve(ids[k:k + c])
            k += c
        assert ((v["action"][:envs] >= 0) & (v["action"][:envs] < num_action)).all()
        for e in range(envs):
            actions[e].append(int(v["action"][e]))
    assert q.get_size() == envs * unrolls
    T = trajectory
    want = {(np.stack(frames[e][u * T:(u + 1) * T]).tobytes(), np.stack(nexts[e][u * T:(u + 1) * T]).tobytes(),
             np.array(actions[e][u * T:(u + 1) * T], np.int32).tobytes())
            for e in range(envs) for u in range(unrolls)}
    got = {(r["state"].tobytes(), r["next_state"].tobytes(), r["action"].tobytes())
           for r in (q.read(j) for j in range(envs * unrolls))}
    assert got == want
    server.close()
    q.close()
    pol.close()
    print("a3c serve loop (cuda graph %s): %d serves of %d environments, %d unrolls committed ok"
          % (graph, unrolls * trajectory + 1, envs, envs * unrolls), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", type=int, nargs="*", default=[2])
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--trajectory", type=int, default=3)
    ap.add_argument("--peer", action="store_true")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--serve", action="store_true", help="the policy server's serve loop instead of learner steps")
    ap.add_argument("--serve-r2d2", action="store_true",
                    help="the R2D2 policy server's serve loop instead of learner steps")
    ap.add_argument("--serve-a3c", action="store_true",
                    help="the A3C policy server's serve loop instead of learner steps")
    a = ap.parse_args()
    if a.serve:
        serve_loop()
        return
    if a.serve_r2d2:
        serve_r2d2_loop()
        return
    if a.serve_a3c:
        serve_a3c_loop()
        return
    from distributed_reinforcement_learning_b200.learner import NativeLearner
    from distributed_reinforcement_learning_b200.model import impala_actor_critic as model
    from oracle import synthetic
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if a.peer:
        import torch
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    for mode in a.modes:
        batch = synthetic.make_batch(a.batch, T=a.trajectory, A=18, seed=5 + rank)
        eng = NativeLearner(batch=a.batch, trajectory=a.trajectory, num_action=18, device=local, math_mode=mode,
                            use_cuda_graph=False)
        eng.set_params(model.init_params(seed=0))
        if a.peer:
            assert eng.enable_peer_exchange()
        for s in range(a.steps):
            eng.stage(s % 2, *[batch[k] for k in synthetic.TRAIN_FIELDS])
            out = eng.step(s % 2)
        assert np.isfinite(out["pi_loss"]) and out["step"] == a.steps
        print("rank %d math_mode %d: %d steps ok, pi_loss %.5f grad_norm %.4f" % (rank, mode, a.steps, out["pi_loss"], out["grad_norm"]),
              flush=True)
        if a.peer:
            dist.barrier()
        eng.close()
    if a.peer:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
