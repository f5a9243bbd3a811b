"""Cases that run every operator UDE kernel (operator.cuh: fixed-step and adaptive Tsit5, fixed-step and adaptive RKC2, forward
and adjoint, fp32 and fp64) through the branches they have: every shape of test_gpu_operator.SHAPES but the two that add no
branch (d = 1, the second lane slot at d = 33, d = 64, D2 = NULL, npde's 30-8-30), the explicit cotangent and the fused L2 with
non-unit loss weights, N = 1, 5 (fewer trajectories than a CTA has warps) and 129 (a partial last CTA), t0 = 0 and t0 != 0,
adaptive solves whose save times fall inside steps, an adaptive RKC2 solve held at its stage cap, and a max_steps failure.
Each case is digested as the sha256 of the bits of out, status, the loss, grad_theta and grad_u0.  Used by
tests/test_gpu_operator_bits.py and tools/make_golden_operator_bits.py."""
import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_operator import ACTN, make  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "operator_bits.json")

SOLVERS = ("tsit5", "tsit5_adaptive", "rkc2", "rkc2_adaptive")
SHAPES = ("d1", "d33_m7", "d64", "d2_null", "npde_30_8_30")
DTYPES = ("float32", "float64")


def _grid():
    """(solver, shape, N, t0, loss path, extra): the product of solvers and shapes, with N, t0 and the cotangent path rotated
    so that each solver sees every value of each; then non-unit loss weights on adaptive Tsit5 (the other solvers meet them at
    d1 or d2_null), the stage cap and the max_steps failure"""
    cases = []
    for i, sv in enumerate(SOLVERS):
        for j, shape in enumerate(SHAPES):
            k = i + j
            cases.append((sv, shape, (1, 5, 129)[k % 3], (0.0, 0.35)[k % 2], ("adjoint", "adjoint_l2")[(k // 2) % 2], ""))
    cases += [("tsit5_adaptive", "d2_null", 129, 0.35, "adjoint_l2", ""),
              ("rkc2_adaptive", "d33_m7", 5, 0.35, "adjoint_l2", "stage_cap"), ("rkc2_adaptive", "npde_30_8_30", 129, 0.0, "adjoint", "stage_cap"),
              ("tsit5_adaptive", "d33_m7", 5, 0.35, "adjoint", "max_steps"), ("rkc2_adaptive", "d64", 5, 0.0, "adjoint_l2", "max_steps")]
    return [c + (dt,) for c in cases for dt in DTYPES]


CASES = _grid()


def key(solver, shape, N, t0, path, extra, dtype):
    return f"{solver},{shape},N={N},t0={t0},{path}" + (f",{extra}" if extra else "") + f",{dtype}"


def solver(solver, shape, N, t0, path, extra, dtype, max_steps=None):
    """the handle of one case and its model, theta and rng (seeded by the shape); max_steps overrides the case's"""
    import torch

    import universal_differential_equations_b200 as ude
    model, theta, rng = make(shape)
    chain = ude.FastChain(*[ude.FastDense(a, b, getattr(ude, ACTN[k])) for a, b, k in zip(model.widths[:-1], model.widths[1:], model.acts)])
    f = ude.OperatorUDE(chain, model.D1, model.D2)
    kw = dict(max_trajectories=N, device="cuda:0", dtype=getattr(torch, dtype))
    if path == "adjoint_l2" and model.d <= 16:   # the operator model takes loss weights up to d = 16
        kw["loss_weights"] = list(rng.uniform(0.2, 2.0, model.d))
    rho = 191.7 if shape == "npde_30_8_30" else 60.0
    if solver == "tsit5":
        return ude.UDESolver(f, t0, 0.05, 12, 2, **kw), model, theta, rng
    if solver == "rkc2":
        return ude.UDESolver(f, t0, 0.05, 12, 3, alg=ude.RKC2(stages=7), **kw), model, theta, rng
    # adaptive: 11 saves 0.04 apart at loose tolerances, so that steps span save times
    kw.update(adaptive=True, abstol=1e-5, reltol=1e-3, max_steps=max_steps or (3 if extra == "max_steps" else 2000))
    if solver == "rkc2_adaptive":
        # stage_cap: 3 stages cannot reach h * eigen_est, so every step is the one the cap allows
        kw["alg"] = ude.RKC2(stages=3, eigen_est=2000.0) if extra == "stage_cap" else ude.RKC2(stages=16, eigen_est=rho)
    return ude.UDESolver(f, t0, 0.04, 10, 1, **kw), model, theta, rng


def run(*case):
    """forward with status, then the case's adjoint: out, status, loss (0 on the explicit cotangent), grad_theta, grad_u0 as numpy"""
    import torch
    s, model, theta, rng = solver(*case)
    N, path, dt = case[2], case[4], s.dtype
    try:
        u0 = rng.normal(scale=0.5, size=(model.d, N))
        n_save = s.n_steps // s.save_every + 1
        s.set_params(torch.tensor(theta, dtype=dt, device="cuda"))
        st = torch.empty(N, dtype=torch.int32, device="cuda")
        out = s.forward(torch.tensor(u0, dtype=dt, device="cuda"), status=st)
        y = torch.tensor(rng.normal(scale=0.5, size=(n_save, model.d, N)), dtype=dt, device="cuda")
        if path == "adjoint_l2":
            loss, g, gu = s.adjoint_l2(y, want_grad_u0=True)
        else:
            (g, gu), loss = s.adjoint(y), torch.zeros(1, dtype=dt)
        torch.cuda.synchronize()
        return out.cpu().numpy(), st.cpu().numpy(), loss.cpu().numpy().reshape(-1), g.cpu().numpy(), gu.cpu().numpy()
    finally:
        s.close()


def status_at(case, max_steps):
    """the forward's status words of an adaptive case solved with at most max_steps accepted steps"""
    import torch
    s, model, theta, rng = solver(*case, max_steps=max_steps)
    try:
        s.set_params(torch.tensor(theta, dtype=s.dtype, device="cuda"))
        st = torch.empty(case[2], dtype=torch.int32, device="cuda")
        s.forward(torch.tensor(rng.normal(scale=0.5, size=(model.d, case[2])), dtype=s.dtype, device="cuda"), status=st)
        return st.cpu().numpy()
    finally:
        s.close()


def bits_digest(out, status, loss, grad_theta, grad_u0):
    h = hashlib.sha256()
    for a in (out, status, loss, grad_theta, grad_u0):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()
