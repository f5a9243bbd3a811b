"""Time one iteration of the SEIR script's call (seir_exposure.jl:137-147: adaptive Vern7 over saveat = 0:21, forward + interpolating
adjoint + fused L2 loss on E, I, R) with Vern7's dense output (B200UDE_FLAG_VERN7_DENSE) and without it (tstops forward, adjoint
over a Tsit5 re-solve).

    python tools/vern7_dense_speed.py [--reps 20] [--rounds 5] [--warmup 3]

fp64 at abstol = reltol = 1e-6 (the script's arithmetic and tolerances); fp32 at 1e-4 (fp32 cannot honour 1e-6 on states of
1.4e7).  N = 1 (the script) and N = 4096.  The two variants run in the same process, alternating: each round times `reps`
back-to-back iterations of one then of the other with CUDA events, after `warmup` untimed iterations of both; the median over
rounds is printed with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import universal_differential_equations_b200 as ude  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _setup(dense, N, dtype, tol, seed=0):
    rng = np.random.default_rng(seed)
    ann = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    theta = ude.initial_params(ann, np.random.default_rng(0))
    u0 = np.tile(np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])[:, None], (1, N))
    u0[2] *= rng.uniform(0.5, 1.5, N)
    solver = ude.UDESolver(ude.SEIRExposureUDE(ann), 0.0, 1.0, 21, 1, max_trajectories=N, alg=ude.Vern7(dense=dense), adaptive=True,
                           abstol=tol, reltol=tol, max_steps=1024, loss_weights=[0, 1, 1, 1, 0, 0, 0], dtype=dtype)
    solver.set_params(torch.as_tensor(theta, dtype=dtype, device="cuda"))
    u = torch.as_tensor(u0, dtype=dtype, device="cuda")
    st = torch.zeros(N, dtype=torch.int32, device="cuda")
    out = solver.forward(u, status=st)
    data = (out * (1 + 0.05 * torch.randn(out.shape, dtype=dtype, device="cuda"))).contiguous()
    gth = torch.empty(solver.P, dtype=dtype, device="cuda")
    loss = torch.empty(1, dtype=dtype, device="cuda")

    def it():
        solver.forward(u, out=out, status=st)
        solver.adjoint_l2(data, grad_theta=gth, loss=loss)
    return solver, it, st


def _time(it, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        it()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, power = _card()
    for dtype, tol in ((torch.float64, 1e-6), (torch.float32, 1e-4)):
        for N in (1, 4096):
            runs = {dense: _setup(dense, N, dtype, tol) for dense in (False, True)}
            for _, it, _ in runs.values():
                for _ in range(a.warmup):
                    it()
            torch.cuda.synchronize()
            ms = {False: [], True: []}
            for _ in range(a.rounds):
                for dense in (False, True):
                    ms[dense].append(_time(runs[dense][1], a.reps))
            ok = all(bool((st == 0).all()) for _, _, st in runs.values())
            print(json.dumps({"case": f"SEIR script call N={N}", "dtype": "f64" if dtype == torch.float64 else "f32", "tol": tol,
                              "tstops_tsit5_resolve_ms": round(float(np.median(ms[False])), 4),
                              "vern7_dense_ms": round(float(np.median(ms[True])), 4),
                              "spread_ms": [round(float(np.ptp(ms[False])), 4), round(float(np.ptp(ms[True])), 4)],
                              "status_ok": ok, "gpu": name, "power_limit": power}), flush=True)
            for s, _, _ in runs.values():
                s.close()


if __name__ == "__main__":
    main()
