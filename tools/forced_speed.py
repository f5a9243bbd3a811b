#!/usr/bin/env python3
"""Time one training iteration of the forced neural ODE (B200UDE_MODEL_FORCED): forward + fused-L2 interpolating adjoint
(b200ude_forward + b200ude_adjoint_l2, reduce included), with CUDA events, fp32 and fp64, for
  - the FENEP.jl script's case: 6 modes, NN pair 2-4-1 / 2-4-1 tanh, Tsit5 adaptive at (1e-6, 1e-3), 100 saves on (0, 6.2831);
  - a sweep of N = 65 536 forcing frequencies (omega in [1, 2]) on the same model.
Prints one JSON line per configuration with the card's name and power limit.  Needs an H100.

Usage:  python tools/forced_speed.py [--iters 50] [--out <file.json>]
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def run(N, dtype, iters):
    f0 = ude.FastChain(ude.FastDense(2, 4, ude.tanh), ude.FastDense(4, 1))
    f1 = ude.FastChain(ude.FastDense(2, 4, ude.tanh), ude.FastDense(4, 1))
    f = ude.ForcedNeuralODE(dynamics=f1, readout=f0)
    rng = np.random.default_rng(0)
    theta = np.concatenate([ude.initial_params(f0, rng), ude.initial_params(f1, rng)])
    t1 = float(np.float32(6.2831))
    s = ude.UDESolver(f, 0.0, t1 / 99, 99, 1, max_trajectories=N, device="cuda:0", adaptive=True, abstol=1e-6, reltol=1e-3,
                      loss_weights=(0.0, 1.0), max_steps=4000, dtype=dtype)
    omega = np.linspace(1.0, 2.0, N)
    s.set_forcing(torch.as_tensor(ude.forcing_coefficients(np.full(N, 12.0), omega), dtype=dtype).cuda())
    s.set_params(torch.as_tensor(theta, dtype=dtype).cuda())
    u0 = torch.zeros((1, N), dtype=dtype, device="cuda")
    data = torch.as_tensor(rng.normal(size=(100, 2, N)), dtype=dtype).cuda()
    out = torch.empty((100, 2, N), dtype=dtype, device="cuda")
    g = torch.empty(s.P, dtype=dtype, device="cuda")
    loss = torch.empty(1, dtype=dtype, device="cuda")
    for _ in range(5):   # warm-up: module load, shape upload, function attributes
        s.forward(u0, out=out)
        s.adjoint_l2(data, grad_theta=g, loss=loss)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = max(1, iters)
    a.record()
    for _ in range(reps):
        s.forward(u0, out=out)
        s.adjoint_l2(data, grad_theta=g, loss=loss)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    return {"N": N, "dtype": str(dtype).replace("torch.", ""), "ms_per_iteration": round(ms, 4), "loss": float(loss)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("forced_speed: needs a CUDA device (no CPU timing is reported)")
    dev = card()
    rows = []
    for N in (6, 65536):
        for dtype in (torch.float32, torch.float64):
            r = run(N, dtype, a.iters if N == 6 else max(5, a.iters // 5))
            r["device"] = dev
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
