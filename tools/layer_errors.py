"""Per-kernel error table of one learner step or one policy-engine act: one JSON line per checked output with the
kernel that wrote it, its per-tensor error, its worst block and the bar it is held to, or its bound ratio
(tests/layer_parity.py for IMPALA, tests/adam_layer_parity.py for Ape-X, A3C and R2D2, tests/policy_layer_parity.py for
the policy engines; the same checks as tests/test_gpu_layer_local.py, tests/test_gpu_adam_layer_local.py and
tests/test_gpu_policy_layer_local.py).  A performance change can show with it which kernel's error moved.

    python tools/layer_errors.py --mode 5 --B 32 --T 20 --A 18 --regime init [--regime trained ...]
    python tools/layer_errors.py --family r2d2 --mode 2 --B 16 --T 80 --burn-in 40 --A 4 --C 1 [--lstm-size 512]
    python tools/layer_errors.py --family apex --mode 2 --B 32 --A 18 [--regime ties]
    python tools/layer_errors.py --family impala_policy --n 64 --A 18 [--regime peaked]
    python tools/layer_errors.py --family r2d2_policy --n 9 --A 4 --C 4 [--regime saturated]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import adam_layer_parity as alp  # noqa: E402
import layer_parity as lp  # noqa: E402
import policy_layer_parity as plp  # noqa: E402

REGIMES = {"impala": lp.REGIMES, "apex": alp.APEX_REGIMES, "a3c": alp.A3C_REGIMES, "r2d2": alp.R2D2_REGIMES}
REGIMES.update({f + "_policy": plp.REGIMES[f] for f in plp.FAMILIES})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--family", choices=sorted(REGIMES), default="impala")
    ap.add_argument("--mode", type=int, default=None, help="math mode (default: 5 for impala, 2 otherwise)")
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=20, help="trajectory (impala) or seq_len (r2d2)")
    ap.add_argument("--burn-in", type=int, default=40, help="r2d2 only")
    ap.add_argument("--A", type=int, default=18)
    ap.add_argument("--C", type=int, default=1, help="r2d2 frame channels")
    ap.add_argument("--lstm-size", type=int, default=64, choices=alp.R2_SIZES, help="r2d2 only")
    ap.add_argument("--n", type=int, default=64, help="rows of the act (policy families)")
    ap.add_argument("--regime", action="append")
    a = ap.parse_args()
    mode = a.mode if a.mode is not None else (5 if a.family == "impala" else 2)
    for r in a.regime or []:
        if r not in REGIMES[a.family]:
            ap.error("regime %r: %s has %s" % (r, a.family, ", ".join(REGIMES[a.family])))
    from distributed_reinforcement_learning_b200 import build
    build.build()
    if a.family.endswith("_policy"):
        fam = a.family[:-len("_policy")]
        C = a.C if fam == "r2d2" else 4
        shape = dict(family=a.family, n=a.n, A=a.A, C=C)
        for regime in a.regime or ["init"]:
            rows, facts = plp.run_case(fam, a.n, a.A, C, regime)
            for r in rows:
                print(json.dumps(dict(shape, regime=regime, **r)), flush=True)
            print(json.dumps(dict(shape, regime=regime, facts=facts)), flush=True)
        return
    shape = dict(family=a.family, mode=mode, B=a.B, A=a.A)
    if a.family in ("impala", "r2d2"):
        shape["T"] = a.T
    if a.family == "r2d2":
        shape.update(burn_in=a.burn_in, C=a.C, lstm_size=a.lstm_size)
    for regime in a.regime or ["init"]:
        if a.family == "impala":
            rows, facts = lp.run_case(mode, a.B, a.T, a.A, regime)
        elif a.family == "r2d2":
            rows, facts = alp.run_r2d2_case(mode, a.B, a.T, a.burn_in, a.A, a.C, regime, L=a.lstm_size)
        else:
            rows, facts = alp.run_apex_case(a.family, mode, a.B, a.A, regime)
        for r in rows:
            print(json.dumps(dict(shape, regime=regime, **r)), flush=True)
        print(json.dumps(dict(shape, regime=regime, facts=facts)), flush=True)


if __name__ == "__main__":
    main()
