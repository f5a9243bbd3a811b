"""Time one training iteration (forward + discrete adjoint + fused L2 loss) of adaptive Vern7 with ForwardDiffSensitivity on the
Fisher-KPP UPDE, beside adaptive Tsit5 with the interpolating adjoint on the same problem (what a script had to use before).

    python tools/fkpp_vern7_discrete_speed.py [--reps 50] [--warmup 5] [--dtype f32|f64]

Cases: scenario_3.jl's problem at N = 1 (26 points, 1-5-5-5-1 rbf, abstol 1e-6 / reltol 1e-3, saveat 0.5 on (0, 5)), N = 4096 on
the same grid, and N = 1024 on a 256-point grid with the 1-16-16-1 tanh chain (D0 = 0.01 / dx^2, t in (0, 0.5)).  CUDA events
around `reps` back-to-back iterations after `warmup` untimed ones; the card's name and power limit are read in the same run.
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


def _chain(widths, act):
    return ude.FastChain(*[ude.FastDense(a, b, act if l < len(widths) - 2 else ude.identity) for l, (a, b) in enumerate(zip(widths[:-1], widths[1:]))])


def _case(Nx, widths, act, N, T, seed=0):
    rng = np.random.default_rng(seed)
    chain = _chain(widths, act)
    theta = np.concatenate([ude.initial_params(chain, rng), [1.0, -2.0, 1.0, 0.0, 0.01 * (Nx - 1) ** 2]])
    x = np.linspace(0.0, 1.0, Nx)[:, None]
    d = rng.uniform(0.2, 0.6, N)[None, :]
    u0 = (np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) / 2
    return ude.FisherKPPUDE(chain, Nx), theta, u0, T


def _time(f, theta, u0, T, alg, sens, dtype, reps, warmup):
    N = u0.shape[1]
    solver = ude.UDESolver(f, 0.0, T / 10, 10, 1, max_trajectories=N, alg=alg, sensealg=sens, adaptive=True, abstol=1e-6, reltol=1e-3,
                           max_steps=2048, dtype=dtype)
    solver.set_params(torch.as_tensor(theta, dtype=dtype, device="cuda"))
    u = torch.as_tensor(u0, dtype=dtype, device="cuda")
    st = torch.zeros(N, dtype=torch.int32, device="cuda")
    out = solver.forward(u, status=st)
    data = (0.9 * out).contiguous()
    gth = torch.empty(solver.P, dtype=dtype, device="cuda")
    loss = torch.empty(1, dtype=dtype, device="cuda")

    def it():
        solver.forward(u, out=out, status=st)
        solver.adjoint_l2(data, grad_theta=gth, loss=loss)
    for _ in range(warmup):
        it()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        it()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    ok = bool((st == 0).all())
    solver.close()
    return ms, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dtype", choices=["f32", "f64"], default="f32")
    a = ap.parse_args()
    dtype = torch.float32 if a.dtype == "f32" else torch.float64
    name, power = _card()
    cases = [("script N=1", _case(26, (1, 5, 5, 5, 1), ude.rbf, 1, 5.0)),
             ("26 pt N=4096", _case(26, (1, 5, 5, 5, 1), ude.rbf, 4096, 5.0)),
             ("256 pt 1-16-16-1 N=1024", _case(256, (1, 16, 16, 1), ude.tanh, 1024, 0.5))]
    for label, (f, theta, u0, T) in cases:
        v7, ok7 = _time(f, theta, u0, T, ude.Vern7(), ude.ForwardDiffSensitivity(), dtype, a.reps, a.warmup)
        ts, okt = _time(f, theta, u0, T, ude.Tsit5(), ude.InterpolatingAdjoint(), dtype, a.reps, a.warmup)
        print(json.dumps({"case": label, "dtype": a.dtype, "vern7_discrete_ms": round(v7, 4), "tsit5_interpolating_ms": round(ts, 4),
                          "status_ok": ok7 and okt, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
