#!/usr/bin/env python3
"""Slice the result files of NonNewtonianFluids/FENEP.jl into tests/golden/fenep.npz.

FENEP.jl:117-123 writes two text files after its training runs:
  plt_data.txt  100 rows `t, sigma_approx_NN, sigma_approx_linear, sigma_exact` for the test strain rate
                gamma_d(t) = 12 cos(1.5 t) at range(0, 10, length = 100);  sigma_exact is its DAE truth (IDA, default tolerances)
  er_data.txt   5000 rows `train_NN, test_NN, train_linear, test_linear`: the errors after every ADAM iteration
Both are guarded by their SHA-256, so a changed reference fails loudly.  Only the numbers go into the npz.

Usage:  python tools/make_golden_fenep.py --ref <reference checkout> [--out tests/golden]
"""
import argparse
import hashlib
import os

import numpy as np

FILES = {
    "plt": ("NonNewtonianFluids/plt_data.txt", "75a745f1fa28bb356dc2db14461df43ced42a696baeb2175b15efb0f64aaa66d"),
    "er": ("NonNewtonianFluids/er_data.txt", "437ef2b05c2e0bc6d6c9701a292e6ee70c4cc2a968df2a1717d37dea53bd69ce"),
}


def load(ref, key):
    rel, sha = FILES[key]
    raw = open(os.path.join(ref, rel), "rb").read()
    got = hashlib.sha256(raw).hexdigest()
    if got != sha:
        raise SystemExit(f"{rel}: sha256 {got} != {sha}")
    return np.loadtxt(raw.decode().splitlines(), delimiter=",")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="checkout of the reference repository")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden"))
    a = ap.parse_args()
    plt = load(a.ref, "plt")
    er = load(a.ref, "er")
    assert plt.shape == (100, 4) and er.shape == (5000, 4)
    np.savez_compressed(os.path.join(a.out, "fenep.npz"), t=plt[:, 0], sigma_nn=plt[:, 1], sigma_linear=plt[:, 2], sigma_exact=plt[:, 3],
                        er_train_nn=er[:, 0].astype(np.float32), er_test_nn=er[:, 1].astype(np.float32),
                        er_train_linear=er[:, 2].astype(np.float32), er_test_linear=er[:, 3].astype(np.float32))
    print("wrote", os.path.join(a.out, "fenep.npz"))


if __name__ == "__main__":
    main()
