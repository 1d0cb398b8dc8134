"""One tiny learner step per math mode for compute-sanitizer (memcheck / racecheck / synccheck of the mbarrier + wgmma
pipelines), and with --peer under torchrun the 2-GPU fused exchange (flag protocol over NVLink peer memory).

    compute-sanitizer --tool memcheck  python tools/sanitize_step.py --modes 2 3
    compute-sanitizer --tool racecheck python tools/sanitize_step.py --modes 2
    torchrun --nproc-per-node 2 ... tools/sanitize_step.py --peer      (run each rank under compute-sanitizer)
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", type=int, nargs="*", default=[2])
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--trajectory", type=int, default=3)
    ap.add_argument("--peer", action="store_true")
    ap.add_argument("--steps", type=int, default=2)
    a = ap.parse_args()
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
