"""Per-kernel error table of one IMPALA learner step: one JSON line per checked output with the kernel that wrote it, its
per-tensor error, its worst block and the bar it is held to (tests/layer_parity.py; the same check as
tests/test_gpu_layer_local.py).  A performance change can show with it which kernel's error moved.

    python tools/layer_errors.py --mode 5 --B 32 --T 20 --A 18 --regime init [--regime trained ...]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import layer_parity as lp  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", type=int, default=5)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=20)
    ap.add_argument("--A", type=int, default=18)
    ap.add_argument("--regime", action="append", choices=lp.REGIMES)
    a = ap.parse_args()
    from distributed_reinforcement_learning_b200 import build
    build.build()
    for regime in a.regime or ["init"]:
        rows, facts = lp.run_case(a.mode, a.B, a.T, a.A, regime)
        for r in rows:
            print(json.dumps(dict(mode=a.mode, B=a.B, T=a.T, A=a.A, regime=regime, **r)), flush=True)
        print(json.dumps(dict(mode=a.mode, B=a.B, T=a.T, A=a.A, regime=regime, facts=facts)), flush=True)


if __name__ == "__main__":
    main()
