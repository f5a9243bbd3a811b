"""Time one training iteration (adaptive Vern7 forward + discrete adjoint + fused L2 loss, ForwardDiffSensitivity) with the save
times as tstops (`Vern7()`) and with free stepping and interpolated saves (`Vern7(dense=True)`, B200UDE_FLAG_DISCRETE_DENSE).

    python tools/vern7_dense_discrete_speed.py [--reps 10] [--rounds 5] [--warmup 3] [--sample 32]

Cases: the LV 2-5-5-5-2 rbf UDE of scenario_1.jl (tspan 0-3, saveat 0.1) at N = 65 536 and the SEIR 3-64-64-1 UDE of
seir_exposure.jl (tspan 0-21, saveat 1, loss on E, I, R) at N = 4096, fp64 and fp32, abstol = reltol = 1e-6 (SEIR in fp32: 1e-4,
fp32 cannot honour 1e-6 on states of 1.4e7).  The two variants run in the same process, alternating: each round times `reps`
back-to-back iterations of one then of the other with CUDA events, after `warmup` untimed iterations of both; the median over
rounds is printed with the card's name and power limit read in the same run.  The mean accepted steps per trajectory of both
variants are counted with the fp64 CPU references of tests/ on the first `sample` trajectories.
"""
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


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _case(form, N, seed=0):
    """(UDE form, oracle model builder, theta, u0[d, N], loss weights, save_dt, n_save)."""
    rng = np.random.default_rng(seed)
    if form == "lv":
        chain = ude.FastChain(*[ude.FastDense(a, b, ude.rbf) for a, b in ((2, 5), (5, 5), (5, 5))], ude.FastDense(5, 2))
        theta = ude.initial_params(chain, np.random.default_rng(1))
        u0 = np.stack([rng.uniform(0.2, 1.0, N), rng.uniform(2.0, 5.0, N)])
        return ude.LotkaVolterraUDE(chain), lambda O: O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity")), theta, u0, [1, 1], 0.1, 31
    ann = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    theta = ude.initial_params(ann, np.random.default_rng(0))
    u0 = np.tile(np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])[:, None], (1, N))
    u0[2] *= rng.uniform(0.5, 1.5, N)
    return ude.SEIRExposureUDE(ann), lambda O: O.seir_model(), theta, u0, [0, 1, 1, 1, 0, 0, 0], 1.0, 22


def _setup(f, theta, u0, w, sdt, ns, dense, dtype, tol):
    N = u0.shape[1]
    solver = ude.UDESolver(f, 0.0, sdt, ns - 1, 1, max_trajectories=N, alg=ude.Vern7(dense=dense), sensealg=ude.ForwardDiffSensitivity(),
                           adaptive=True, abstol=tol, reltol=tol, max_steps=1024, loss_weights=w, dtype=dtype)
    solver.set_params(torch.as_tensor(theta, dtype=dtype, device="cuda"))
    u = torch.as_tensor(u0, dtype=dtype, device="cuda")
    st = torch.zeros(N, dtype=torch.int32, device="cuda")
    out = solver.forward(u, status=st)
    data = (out * (1 + 0.05 * torch.randn(out.shape, dtype=dtype, device="cuda", generator=torch.Generator("cuda").manual_seed(0)))).contiguous()
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


def _mean_steps(model_of, theta, u0, sdt, ns, tol, sample):
    """Mean accepted steps (tstops, free stepping) of the fp64 CPU references over the first `sample` trajectories."""
    import discrete_ref
    import vern7_dense_ref
    from oracle import oracle as O
    O.build()
    m = model_of(O)
    th = np.asarray(theta, np.float64)
    k = min(sample, u0.shape[1])
    a = [len(discrete_ref.vern7_adaptive_record(O, m, th, u0[:, i], 0.0, sdt, ns, tol, tol)[1]["hstep"]) for i in range(k)]
    b = [len(vern7_dense_ref.dense_record(O, m, th, u0[:, i], 0.0, sdt, ns, tol, tol)[1]["hstep"]) for i in range(k)]
    return float(np.mean(a)), float(np.mean(b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=32)
    ap.add_argument("--n-lv", type=int, default=65536)
    ap.add_argument("--n-seir", type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, power = _card()
    for form, N in (("lv", a.n_lv), ("seir", a.n_seir)):
        f, model_of, theta, u0, w, sdt, ns = _case(form, N)
        for dtype in (torch.float64, torch.float32):
            tol = 1e-4 if (form == "seir" and dtype == torch.float32) else 1e-6
            steps = _mean_steps(model_of, theta, u0, sdt, ns, tol, a.sample)
            runs = {dense: _setup(f, theta, u0, w, sdt, ns, dense, dtype, tol) for dense in (False, True)}
            for _, it, _ in runs.values():
                for _ in range(a.warmup):
                    it()
            torch.cuda.synchronize()
            ms = {False: [], True: []}
            for _ in range(a.rounds):
                for dense in (False, True):
                    ms[dense].append(_time(runs[dense][1], a.reps))
            ok = all(bool((st == 0).all()) for _, _, st in runs.values())
            print(json.dumps({"case": f"{form} N={N}", "dtype": "f64" if dtype == torch.float64 else "f32", "tol": tol,
                              "tstops_discrete_ms": round(float(np.median(ms[False])), 4),
                              "dense_discrete_ms": round(float(np.median(ms[True])), 4),
                              "spread_ms": [round(float(np.ptp(ms[False])), 4), round(float(np.ptp(ms[True])), 4)],
                              "mean_accepted_steps_fp64_ref": {"tstops": round(steps[0], 2), "dense": round(steps[1], 2), "sample": min(a.sample, N)},
                              "status_ok": ok, "gpu": name, "power_limit": power}), flush=True)
            for s, _, _ in runs.values():
                s.close()


if __name__ == "__main__":
    main()
