"""Time one training iteration of the operator UDE (npde.jl's 30-8-30 tanh closure): forward, fused-L2 adjoint and reduce.

Fixed-step Tsit5 at a quarter of the save spacing (h rho(D2) = 2.5 for npde's rho = 191.7, inside Tsit5's real stability
interval of about 3.5), adaptive Tsit5 at
(1e-6, 1e-3), fixed-step RKC2 at the save spacing with the stage count from eigen_est = rho(D2), and adaptive RKC2 at
(1e-6, 1e-3) with the stage count of each step from eigen_est, fp32 and fp64, for N = 1 (the script's case) and
ensembles of initial bumps; then the forward of the t = 10 solve (npde.jl:120-123: adaptive, (1e-4, 1e-2), save grid 10/194),
adaptive RKC2 against adaptive Tsit5.  CUDA events; the configurations alternate
round by round, and the median and the spread over rounds are printed with the GPU's name and power limit.
Usage: python tools/operator_speed.py [--rounds 7] [--iters 20] [--sizes 1,4096,65536]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import universal_differential_equations_b200 as ude  # noqa: E402
import operator_ref as R  # noqa: E402


def bumps(N, rng):
    z = R.npde_grid()[1:31]
    c = rng.uniform(0.2, 0.8, N) if N > 1 else np.array([0.75])
    return np.exp(-200.0 * (z[:, None] - c[None, :]) ** 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sizes", default="1,4096,65536")
    a = ap.parse_args()
    D1, D2 = R.npde_ops()
    saveat = np.linspace(0, 1.5, 30)
    chain = ude.FastChain(ude.FastDense(30, 8, ude.tanh), ude.FastDense(8, 30, ude.tanh))
    f = ude.OperatorUDE(chain, D1, D2)
    th = R.glorot([30, 8, 30], np.random.default_rng(0))
    stages = ude.RKC2(eigen_est=191.7).n_stages(saveat[1])
    n10 = int(np.ceil(10.0 / saveat[1]))

    def make(N, dt, solver, t10=False):
        kw = {"tsit5": {}, "tsit5_adaptive": dict(adaptive=True), "rkc2": dict(alg=ude.RKC2(stages=stages)),
              "rkc2_adaptive": dict(alg=ude.RKC2(eigen_est=191.7), adaptive=True)}[solver]
        if t10:   # npde.jl:120-123: the forward of the t = 10 solve at (1e-4, 1e-2) on the save grid 10/194
            s = ude.UDESolver(f, 0.0, 10.0 / n10, n10, 1, max_trajectories=1, device="cuda:0", dtype=dt, abstol=1e-4, reltol=1e-2,
                              max_steps=2000, **kw)
        elif solver == "tsit5":
            s = ude.UDESolver(f, 0.0, saveat[1] / 4, 29 * 4, 4, max_trajectories=N, device="cuda:0", dtype=dt)
        else:
            s = ude.UDESolver(f, 0.0, saveat[1], 29, 1, max_trajectories=N, device="cuda:0", dtype=dt, abstol=1e-6, reltol=1e-3,
                              max_steps=400, **kw)
        s.set_params(torch.tensor(th, dtype=dt, device="cuda"))
        u = torch.tensor(bumps(N, np.random.default_rng(N)), dtype=dt, device="cuda")   # the same bumps for every solver
        data = None if t10 else (s.forward(u) * 1.01).contiguous()
        return dict(N=N, dtype=str(dt).split(".")[-1], solver=solver + ("_t10_forward" if t10 else ""), s=s, u=u, data=data, times=[])

    def step(c):
        c["s"].forward(c["u"])
        if c["data"] is not None:
            c["s"].adjoint_l2(c["data"])

    # one group per ensemble size and dtype (at N = 65 536 the records of all eight do not fit the device at once); the
    # configurations of a group alternate round by round
    dts = (torch.float32, torch.float64)
    groups = [[(N, dt, sv, False) for sv in ("tsit5", "tsit5_adaptive", "rkc2", "rkc2_adaptive")] for N in [int(x) for x in a.sizes.split(",")] for dt in dts]
    groups.append([(1, dt, sv, True) for dt in dts for sv in ("tsit5_adaptive", "rkc2_adaptive")])
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# GPU: {q}; fixed-step RKC2 stages = {stages}; ms per iteration (forward + fused-L2 adjoint + reduce; *_t10_forward: "
          f"the forward alone), median [min, max] over {a.rounds} rounds")
    for g in groups:
        cfgs = [make(*x) for x in g]
        for c in cfgs:   # warm-up
            for _ in range(3):
                step(c)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for c in cfgs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    step(c)
                e1.record()
                e1.synchronize()
                c["times"].append(e0.elapsed_time(e1) / a.iters)
        for c in cfgs:
            t = np.array(c["times"])
            print(json.dumps(dict(N=c["N"], dtype=c["dtype"], solver=c["solver"], ms_median=round(float(np.median(t)), 4),
                                  ms_min=round(float(t.min()), 4), ms_max=round(float(t.max()), 4))), flush=True)
            c["s"].close()
        del cfgs
        torch.cuda.empty_cache()

if __name__ == "__main__":
    main()
