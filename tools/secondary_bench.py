#!/usr/bin/env python3
"""Secondary workloads of SURVEY.md section 8(d) -- BASELINE configs 3 (SEIR exposure UDE) and 4 (Fisher-KPP UPDE) and the
adaptive / Vern7 paths -- measured like bench.py's headline: CUDA events around K steps after W warm-ups, inputs resident
in HBM, the CPU oracle port timed beside on a bounded sample.  One JSON line per workload (not the driver's bench line).

  python tools/secondary_bench.py [--steps K] [--warmup W] [--no-cpu]
"""
import argparse, json, os, sys, time
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import universal_differential_equations_b200 as ude
from helpers import glorot_theta, synthetic_ensemble

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5); ap.add_argument("--warmup", type=int, default=3); ap.add_argument("--no-cpu", action="store_true")
args = ap.parse_args()
FP32_PEAK = 72.5e12


def gpu_time(solver, theta, u0, y):
    th = torch.from_numpy(theta).cuda(); u0d = torch.from_numpy(u0).cuda(); yd = torch.from_numpy(y).cuda()
    solver.set_params(th)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tf = ta = 0.0
    for it in range(args.warmup + args.steps):
        flush.zero_()
        ev[0].record(); solver.forward(u0d); ev[1].record(); solver.adjoint_l2(yd); ev[2].record(); torch.cuda.synchronize()
        if it >= args.warmup:
            tf += ev[0].elapsed_time(ev[1]) / args.steps; ta += ev[1].elapsed_time(ev[2]) / args.steps
    return tf, ta


def cpu_rate(model, theta, u0, y, w, dt, n_steps, every, sample):
    if args.no_cpu:
        return None
    from oracle import oracle as O
    t = time.perf_counter()
    O.ensemble_loss_grad(model, theta.astype(np.float32), u0[:, :sample], y[:, :, :sample], np.asarray(w, np.float32), dt, n_steps, save_every=every, want_gu0=False)
    return sample / (time.perf_counter() - t)


def report(name, N, tf, ta, flop, cpu, extra):
    rate = N / ((tf + ta) * 1e-3)
    line = {"workload": name, "metric": "ensemble trajectories/sec fwd+adjoint", "value": rate, "unit": "trajectories/s", "n_gpus": 1,
            "trajectories": N, "fwd_ms": tf, "adj_ms": ta, "dtype": "f32", "data": "synthetic",
            "roofline_fp32": {"bound": "fp32", "achieved": flop * rate / 1e12, "peak": FP32_PEAK / 1e12, "unit": "TFLOP/s", "frac": flop * rate / FP32_PEAK},
            "cpu_baseline": None if cpu is None else {"value": cpu, "unit": "trajectories/s", "cores": os.cpu_count(), "kind": "port"}}
    line.update(extra)
    print(json.dumps(line), flush=True)


rng = np.random.default_rng(0)
# ---- config 3: SEIR exposure UDE, reference shape (7 states, 3-64-64-1), Tsit5 dt = 0.25 x 84 (tspan (0, 21)), saved daily, loss on E, I, R
N = 65536
chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
theta = glorot_theta((3, 64, 64, 1), seed=2)
S0 = 14e6
u0 = np.zeros((7, N), np.float32); u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N); u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = S0
y = rng.uniform(0, 100, (22, 7, N)).astype(np.float32)
w = [0, 1, 1, 1, 0, 0, 0]
s = ude.UDESolver(ude.SEIRExposureUDE(chain), 0.0, 0.25, 84, 4, max_trajectories=N, loss_weights=w)
tf, ta = gpu_time(s, theta, u0, y)
s.close()
fma = 3 * 64 + 64 * 64 + 64
flop = 2.0 * fma * (1 + 6 * 84) + 2.0 * 3 * fma * 6 * 84
from oracle import oracle as O
cpu = cpu_rate(O.seir_model(), theta, u0, y, w, 0.25, 84, 4, 2048)
report("SEIR exposure UDE 7-state 3-64-64-1, Tsit5 dt=0.25 x84, N=65536 (BASELINE config 3, reference shape)", N, tf, ta, flop, cpu,
       {"kernels": "seir::forward_kernel / seir::adjoint_kernel (3xTF32 mma.sync)", "flop_per_trajectory": flop})

# ---- config 4: Fisher-KPP UPDE, 256-point grid, 1-16-16-1 tanh reaction chain + 3-tap periodic stencil, Tsit5
Nx, N = 256, 8192
widths = (1, 16, 16, 1)
layers = [ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)]
f = ude.FisherKPPUDE(ude.FastChain(*layers), Nx)
D0 = 0.01 * (Nx - 1) ** 2                       # D / dx^2 with the reference's D = 0.01 (Fisher-KPP-CNN.jl:16-25)
theta = np.concatenate([glorot_theta(widths, seed=3), [1.0, -2.0, 1.0, 0.0, D0]]).astype(np.float32)
x = np.linspace(0, 1, Nx)
u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) for d in rng.uniform(0.15, 0.5, N)], axis=1).astype(np.float32)
n_steps, every = 200, 20
dtv = 1.0e-3                                    # explicit-RK stability: dt * 4 D0 < ~3.3
y = np.repeat(u0[None], n_steps // every + 1, axis=0)
s = ude.UDESolver(f, 0.0, dtv, n_steps, every, max_trajectories=N)
tf, ta = gpu_time(s, theta, u0, y)
s.close()
fma = Nx * (16 + 256 + 16 + 4)
flop = 2.0 * fma * (1 + 6 * n_steps) + 2.0 * 3 * fma * 6 * n_steps
cpu = cpu_rate(O.fkpp_model(Nx, widths, ("tanh", "tanh", "identity")), theta, u0, y, np.ones(Nx), dtv, n_steps, every, 256)
report("Fisher-KPP UPDE 256-point grid, 1-16-16-1 + 3-tap stencil, Tsit5 dt=1e-3 x200, N=8192 (BASELINE config 4 shape, Tsit5 instead of ROCK2)", N, tf, ta, flop, cpu,
       {"kernels": "fkpp kernels", "flop_per_trajectory": flop, "grid_points_per_s": N * Nx / ((tf + ta) * 1e-3)})

# ---- adaptive Tsit5 (abstol = reltol = 1e-6) on the headline chain
N = 65536
chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
theta = glorot_theta((2, 32, 32, 2), seed=1)
u0, y = synthetic_ensemble(N)
s = ude.UDESolver(ude.LotkaVolterraUDE(chain), 0.0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=1e-6, reltol=1e-6, max_steps=128)
tf, ta = gpu_time(s, theta, u0, y)
s.close()
report("LV 2-32-32-2 ADAPTIVE Tsit5 abstol=reltol=1e-6, N=65536", N, tf, ta, 0.0, None, {"kernels": "lv32::tc::adaptive_forward_kernel / lv32::tc::adjoint_kernel<ADAPT> (B200UDE_ADAPTIVE_TC=0: generic::adaptive_*<Ops32, 128>)"})

# ---- SEIR exposure UDE, adaptive Tsit5 abstol = reltol = 1e-4 (fp32 states of magnitude 1e7), saved daily
N = 65536
chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
theta = glorot_theta((3, 64, 64, 1), seed=2)
u0 = np.zeros((7, N), np.float32); u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N); u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = S0
y = rng.uniform(0, 100, (22, 7, N)).astype(np.float32)
s = ude.UDESolver(ude.SEIRExposureUDE(chain), 0.0, 1.0, 21, 1, max_trajectories=N, loss_weights=[0, 1, 1, 1, 0, 0, 0], adaptive=True, abstol=1e-4, reltol=1e-4, max_steps=128)
tf, ta = gpu_time(s, theta, u0, y)
s.close()
report("SEIR exposure UDE 3-64-64-1 ADAPTIVE Tsit5 abstol=reltol=1e-4, saveat daily over (0, 21), N=65536", N, tf, ta, 0.0, None, {"kernels": "seir::adaptive_forward_kernel / seir::adjoint_kernel<ADAPT>"})
