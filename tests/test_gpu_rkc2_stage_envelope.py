"""RKC2 at every stage count the handles accept (2 <= s <= 64), on the GPU.

- Operator UDE, fixed step (operator.cuh kernels 5 and 6), fp64 and fp32: a linear closure whose RKC2 solution and dL/du0 are
  closed-form (rkc2_closed_form.py, mpmath), with a stiff spectrum spread over the whole stability interval of each s; plus the
  npde 30-8-30 tanh closure at a few s against operator_ref.py.
- Operator UDE, adaptive RKC2 (kernels 7 and 8): eigen_est values that together select every stage count 2..64, the capped
  branch (beta(cap) < 1.05 h eigen_est), and fp32 at high stage counts.
- Fisher-KPP packed kernels (fkpp_tuned.cuh forward_rkc_kernel2 / adjoint_kernel2<.., true>), fp32: zero reaction against the
  closed-form Fourier solution, and the 1-16-16-1 tanh reaction against the fp64 oracle.

fp32 states and dL/du0 are held to 2e-5 (1 + |x|) at every s, fp64 to 1e-12 of the solution's scale.  The stiff part of the
linear closure is diagonal, so rounding f = M u puts each stiff component's error on that (damped) component; what these bounds
see is the round-off of the stage recurrence itself, which the kernels keep small by carrying the increments Y_j - u."""
import functools
import os
import sys

import mpmath as mp
import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import operator_ref as R  # noqa: E402
import operator_rkc2_adaptive_ref as A  # noqa: E402
import rkc2_closed_form as CF  # noqa: E402
from helpers import glorot_theta  # noqa: E402
from test_gpu_operator import make, rel, run, solver_for  # noqa: E402

pytestmark = pytest.mark.gpu

STAGES = list(range(2, 65))
D, M = 33, 7                       # two state components per lane on the lanes 0 and 1; m = 7 outputs of the closure
H, N_STEPS, EVERY, NTRAJ = 0.05, 100, 10, 3


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


# ---------------------------------------------------------------- operator, fixed step, linear closure
@functools.lru_cache(maxsize=None)
def linear_case(s):
    """du = D1 (W u + b) + D2 u with every input exactly representable in fp32 (so the fp32 and fp64 handles see the same
    problem), W = c D1^T with c a power of two so that M = D1 W + D2 is symmetric; D2 diagonal with its entries spread
    log-uniformly over [1e-3, 0.9 beta(s)] / h.  A diagonal D2 keeps the rounding of a stiff component of f on that component,
    which the stability polynomial damps; a dense one would spread it onto the slow modes, where it is not damped and would
    hide the recurrence's own round-off.  Returns the inputs, theta, u0, the cotangents and the closed-form saves and dL/du0."""
    rng = np.random.default_rng(1000 + s)
    beta = float(CF.Rkc2(s).beta)
    D1 = f32(rng.normal(scale=1.0 / np.sqrt(M), size=(D, M)))
    c = 2.0 ** np.floor(np.log2(5e-4 / (H * np.linalg.norm(D1, 2) ** 2)))   # h ||D1 W|| <= 5e-4: D1 W moves no eigenvalue past 0
    W = c * D1.T
    b = f32(rng.normal(scale=0.1, size=M))
    D2 = np.diag(f32(-rng.permutation(np.geomspace(1e-3, 0.9 * beta, D)) / H))
    Mx = D1 @ W + D2
    Mx = (Mx + Mx.T) / 2
    with mp.workdps(CF.DPS):
        E, V = mp.eigsy(mp.matrix((H * Mx).tolist()))
        hl = np.array([float(e) for e in E])
        V = np.array([[float(V[i, j]) for j in range(D)] for i in range(D)])
        rk = CF.Rkc2(s)
        p = [rk.P(mp.mpf(float(e))) for e in E]
        # P_s(hM)^k (k = 0, EVERY, ..) and the affine part of the augmented step map, sum_{i<k} P^i (P - 1) / (hM) h D1 b
        pk = [np.array([float(v ** k) for v in p]) for k in range(0, N_STEPS + 1, EVERY)]
        ak = [np.array([float((v ** k - 1) / mp.mpf(float(e))) for v, e in zip(p, E)]) for k in range(0, N_STEPS + 1, EVERY)]
    assert (hl >= -0.95 * beta).all() and (hl < 0).all(), (hl.min(), hl.max(), beta)
    assert max(abs(x) for x in pk[1]) < 1.0
    u0 = f32(V @ (rng.uniform(0.5, 1.5, size=(D, NTRAJ)) * rng.choice([-1.0, 1.0], size=(D, NTRAJ))))   # O(1) on every eigenvector
    cot = f32(rng.normal(size=(N_STEPS // EVERY + 1, D, NTRAJ)))
    g = H * (D1 @ b)
    Vg = V.T @ g
    out = np.array([V @ (q[:, None] * (V.T @ u0)) + (V @ (a * Vg))[:, None] for q, a in zip(pk, ak)])
    gu0 = sum(V @ (q[:, None] * (V.T @ ck)) for q, ck in zip(pk, cot))
    theta = np.concatenate([W.T.ravel(), b])   # vec(W) column-major, then b
    model = R.Model((D, M), (0,), D1, D2)
    return model, theta, u0, cot, out, gu0


@pytest.mark.parametrize("s", STAGES)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_fixed_step_linear_closure_vs_closed_form(s, dtype):
    import universal_differential_equations_b200 as ude
    model, theta, u0, cot, ref, gref = linear_case(s)
    sv = solver_for(model, dtype, NTRAJ, H, N_STEPS, EVERY, alg=ude.RKC2(stages=s))
    out, st, _, g, gu = run(sv, theta, u0, cot=cot)
    assert (st == 0).all()
    eo, eg = np.abs(out - ref), np.abs(gu - gref)
    if dtype == torch.float64:
        so, sg = max(1.0, np.abs(ref).max()), max(1.0, np.abs(gref).max())
        print(f"MEASURED fp64 RKC2 s = {s}, {N_STEPS} steps: state {eo.max() / so:.2e}, dL/du0 {eg.max() / sg:.2e} (relative to scale)")
        assert eo.max() <= 1e-12 * so and eg.max() <= 1e-12 * sg, (s, eo.max() / so, eg.max() / sg)
        gth = np.zeros(model.P)
        for j in range(NTRAJ):
            _, rec = R.rkc2_fixed(model, theta, u0[:, j], H, N_STEPS, s, EVERY)
            gth += R.rkc2_adjoint(model, theta, rec, H, N_STEPS, s, EVERY, cot[:, :, j])[0]
        assert rel(g, gth) <= 1e-10, (s, rel(g, gth))
    else:
        ro, rg = (eo / (1 + np.abs(ref))).max(), (eg / (1 + np.abs(gref))).max()
        print(f"MEASURED fp32 RKC2 s = {s}, {N_STEPS} steps: state {ro:.2e}, dL/du0 {rg:.2e} (relative to 1 + |x|)")
        assert ro <= 2e-5 and rg <= 2e-5, (s, ro, rg)


@pytest.mark.parametrize("s", [2, 3, 17, 64])
def test_fixed_step_npde_closure_vs_reference(s):
    import universal_differential_equations_b200 as ude
    model, theta, rng = make("npde_30_8_30")
    rho = np.abs(np.linalg.eigvalsh(model.D2)).max() + np.linalg.norm(model.D1, 2) * np.prod(
        [np.linalg.norm(W, 2) for W, _, _, _ in model.layers(theta)])
    dt = min(0.5 * A.beta(s) / rho, 0.2)
    n, every = 20, 2
    u0 = rng.normal(scale=0.5, size=(model.d, NTRAJ))
    cot = rng.normal(size=(n // every + 1, model.d, NTRAJ))
    out, st, _, g, gu = run(solver_for(model, torch.float64, NTRAJ, dt, n, every, alg=ude.RKC2(stages=s)), theta, u0, cot=cot)
    assert (st == 0).all()
    gref = np.zeros(model.P)
    for j in range(NTRAJ):
        o, rec = R.rkc2_fixed(model, theta, u0[:, j], dt, n, s, every)
        gt, lam, _ = R.rkc2_adjoint(model, theta, rec, dt, n, s, every, cot[:, :, j])
        gref += gt
        assert rel(out[:, :, j], o) < 1e-10 and rel(gu[:, j], lam) < 1e-10
    assert rel(g, gref) < 1e-10


# ---------------------------------------------------------------- operator, adaptive RKC2
SAVE_DT, N_SAVE, TOL = 0.1, 11, (1e-6, 1e-3)
# eigen_est values from s = 2 on every step up to steps at the 64-stage cap; together they select every stage count 2..64
RHOS = [2.0, 30.0, 120.0, 400.0, 1200.0, 3000.0, 7000.0, 15000.0, 30000.0, 60000.0, 120000.0, 250000.0]


def adaptive(model, dtype, N, rho, stages=None, max_steps=4000):
    import universal_differential_equations_b200 as ude
    return solver_for(model, dtype, N, SAVE_DT, N_SAVE - 1, 1, alg=ude.RKC2(stages=stages, eigen_est=rho), adaptive=True,
                      abstol=TOL[0], reltol=TOL[1], max_steps=max_steps)


@functools.lru_cache(maxsize=None)
def adaptive_case(rho, cap=64):
    model, theta, rng = make("npde_30_8_30")
    u0 = rng.normal(scale=0.5, size=(model.d, NTRAJ))
    cot = rng.normal(size=(N_SAVE, model.d, NTRAJ))
    refs = []
    for j in range(NTRAJ):
        o, rec, stj = A.rkc2_adaptive(model, theta, u0[:, j], 0.0, SAVE_DT, N_SAVE, TOL[0], TOL[1], rho, cap=cap)
        assert stj == 0
        refs.append((o, rec, A.rkc2_adaptive_adjoint(model, theta, rec, 0.0, SAVE_DT, N_SAVE, o, cot[:, :, j])))
    return model, theta, u0, cot, refs


def check_fp64_against_reference(rho, cap=64):
    model, theta, u0, cot, refs = adaptive_case(rho, cap)
    stages = None if cap == 64 else cap
    out, st, _, g, gu = run(adaptive(model, torch.float64, NTRAJ, rho, stages), theta, u0, cot=cot)
    assert (st == 0).all()
    for j, (o, rec, (_, lam, _)) in enumerate(refs):
        assert rel(out[:, :, j], o) < 1e-9 and rel(gu[:, j], lam) < 1e-9, (rho, cap, j)
    assert rel(g, sum(r[2][0] for r in refs)) < 1e-9
    # the kernel's accepted-step count of trajectory 0 is the reference's: max_steps = n - 1 fails (status 2), n succeeds
    n = len(refs[0][1][3])
    for ms in (n - 1, n):
        st = run(adaptive(model, torch.float64, 1, rho, stages, max_steps=ms), theta, u0[:, :1], cot=cot[:, :, :1])[1]
        assert st[0] == (2 if ms < n else 0), (rho, cap, ms, n)


def test_adaptive_eigen_est_values_cover_every_stage_count():
    used = set()
    for rho in RHOS:
        used |= {s for _, rec, _ in adaptive_case(rho)[4] for s in rec[3]}
    print(f"adaptive RKC2 stage counts used over eigen_est {RHOS}: {sorted(used)}")
    assert used == set(range(2, 65)), sorted(set(range(2, 65)) - used)
    assert set(adaptive_case(RHOS[0])[4][0][1][3]) == {2}


@pytest.mark.parametrize("rho", RHOS)
def test_adaptive_fp64_matches_reference_at_every_stage_count(rho):
    check_fp64_against_reference(rho)


@pytest.mark.parametrize("cap", [2, 3, 4, 17])
def test_adaptive_capped_stage_count(cap):
    """eigen_est so large that beta(cap) < 1.05 h eigen_est on most steps: those steps take h = beta(cap) / (1.05 eigen_est)."""
    rho = 100.0 * A.beta(cap)
    _, _, _, _, refs = adaptive_case(rho, cap)
    for _, rec, _ in refs:
        h, s = np.diff(rec[2]), np.array(rec[3])
        capped = (s == cap) & (np.abs(h - A.beta(cap) / (1.05 * rho)) <= 1e-12 * h)
        assert capped.mean() > 0.5, (cap, capped.mean())
    check_fp64_against_reference(rho, cap)


def test_adaptive_fp32_at_high_stage_counts():
    rho = next(r for r in RHOS if min(adaptive_case(r)[4][0][1][3][2:]) >= 40)
    model, theta, u0, cot, refs = adaptive_case(rho)
    th32, u32 = f32(theta), f32(u0)
    data = f32(np.random.default_rng(5).normal(scale=0.5, size=(N_SAVE, model.d, NTRAJ)))
    out, st, loss, g, gu = run(adaptive(model, torch.float32, NTRAJ, rho, max_steps=400), th32, u32, data=data)
    assert (st == 0).all()
    gref, lref = np.zeros(model.P), 0.0
    for j in range(NTRAJ):
        o, rec, stj = A.rkc2_adaptive(model, th32, u32[:, j], 0.0, SAVE_DT, N_SAVE, TOL[0], TOL[1], rho)
        assert stj == 0 and len(rec[3]) < 400
        gt, lam, l = A.rkc2_adaptive_adjoint(model, th32, rec, 0.0, SAVE_DT, N_SAVE, o, data[:, :, j], fused=True)
        gref += gt
        lref += l
        print(f"MEASURED fp32 adaptive RKC2 eigen_est {rho}: stages {min(rec[3])}..{max(rec[3])}, state {rel(out[:, :, j], o):.2e}, "
              f"dL/du0 {rel(gu[:, j], lam):.2e}")
        assert rel(out[:, :, j], o) < 2e-5 and rel(gu[:, j], lam) < 1e-3
    assert abs(loss - lref) / lref < 1e-4 and rel(g, gref) < 1e-3


# ---------------------------------------------------------------- Fisher-KPP packed kernels, fp32
FK_WIDTHS = (1, 16, 16, 1)


def fkpp_solver(nx, N, dt, n_steps, every, s):
    import universal_differential_equations_b200 as ude
    layers = [ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)]
    return ude.UDESolver(ude.FisherKPPUDE(ude.FastChain(*layers), nx), 0.0, dt, n_steps, every, max_trajectories=N,
                         alg=ude.ROCK2(stages=s))


@pytest.mark.parametrize("s", [2, 3, 16, 33, 64])
@pytest.mark.parametrize("nx", [64, 256])
@pytest.mark.parametrize("asym", [False, True])
def test_fkpp_zero_reaction_vs_closed_form(s, nx, asym):
    """the reaction network's last layer is zero, so du = D0 (w1 u_{i-1} + w2 u_i + w3 u_{i+1}): each Fourier mode is multiplied
    by P_s(h lambda_k) per step, h = 0.95 beta(s) / rho.  Bound 2e-5 (1 + |x|) for states and dL/du0.

    The asymmetric stencil at s >= 33 cannot meet it in fp32 however the stages are ordered.  Its weights 1 +- delta need more
    mantissa bits than a float has, so each evaluation of f rounds by ~eps |u| D0 on every point, and a step multiplies that by
    h D0 = 0.95 beta(s) / 4 (170 at s = 33, 635 at s = 64).  The error is as smooth as u, so it lands on the slow modes that the
    step does not damp.  With weights (1, -2, 1), and the positive, smooth u and cotangents used here, the stencil's products and
    first sum are exact.  Those cases are held to 1e-4.  Measured on an H100 (80 GB, 700 W), largest over both grids: symmetric,
    states 7.1e-6 and dL/du0 5.8e-6 at s = 64; asymmetric, states 3.8e-5 at s = 64 and dL/du0 4.1e-5 at s = 33."""
    rng = np.random.default_rng(nx + s)
    D0 = 0.01 * (nx - 1) ** 2
    rk = CF.Rkc2(s)
    h = 0.95 * float(rk.beta) / (4 * D0)
    # the asymmetric stencil's imaginary spectrum, 2 delta D0 h, stays inside the thin stability region around the real axis
    # (a power of two, so that w1 + w2 + w3 = 0 in fp32 too and the constant mode is kept exactly)
    delta = 2.0 ** np.floor(np.log2(min(0.05, 0.25 / (D0 * h)))) if asym else 0.0
    w = (1.0 + delta, -2.0, 1.0 - delta)
    theta = glorot_theta(FK_WIDTHS, seed=3)
    theta[-17:] = 0.0                                    # last layer W3 (16) and b3: the reaction output is exactly 0
    theta = np.concatenate([theta, [*w, 0.0, D0]]).astype(np.float32)
    stencil = tuple(float(np.float32(v)) for v in (*w, D0))
    lam = CF.stencil_symbol(nx, *stencil)
    with mp.workdps(CF.DPS):
        amp = [abs(rk.P(mp.mpc(h * complex(l)))) for l in lam]
        assert lam[0] == 0 and amp[0] == 1 and all(a < 1 for a in amp[1:]), float(max(amp[1:]))
    N, n_steps, every = 3, 100, 10
    x = np.arange(nx) / nx
    u0 = f32(np.stack([0.5 + 0.3 * np.sin(2 * np.pi * (x + p)) + 0.05 * rng.normal(size=nx) for p in rng.uniform(0, 1, N)], axis=1))
    # positive, smooth cotangents (a weighted mean of the state at each save), so that lambda stays positive and smooth like u
    cot = f32(0.5 + 0.3 * np.sin(2 * np.pi * (x[None, :, None] + rng.uniform(0, 1, (n_steps // every + 1, 1, N)))))
    sv = fkpp_solver(nx, N, np.float32(h), n_steps, every, s)
    sv.set_params(torch.from_numpy(theta).cuda())
    st = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = sv.forward(torch.from_numpy(u0.astype(np.float32)).cuda(), status=st)
    _, gu = sv.adjoint(torch.from_numpy(cot.astype(np.float32)).cuda())
    torch.cuda.synchronize()
    out, gu, st = out.cpu().numpy().astype(np.float64), gu.cpu().numpy().astype(np.float64), st.cpu().numpy()
    sv.close()
    assert (st == 0).all()
    hh = float(np.float32(h))
    worst_o = worst_g = 0.0
    for k in range(N):
        ref = CF.periodic_diffusion_solution(u0[:, k], stencil, hh, s, n_steps, every)
        gref = CF.periodic_diffusion_grad_u0(cot[:, :, k], stencil, hh, s, n_steps, every)
        worst_o = max(worst_o, (np.abs(out[:, :, k] - ref) / (1 + np.abs(ref))).max())
        worst_g = max(worst_g, (np.abs(gu[:, k] - gref) / (1 + np.abs(gref))).max())
    tol = 1e-4 if asym and s >= 33 else 2e-5
    print(f"MEASURED fp32 Fisher-KPP zero reaction s = {s}, nx = {nx}, delta = {delta:.3g}: state {worst_o:.2e}, dL/du0 {worst_g:.2e}")
    assert worst_o <= tol and worst_g <= tol, (worst_o, worst_g, tol)


@pytest.mark.parametrize("s", [2, 16, 64])
def test_fkpp_tanh_reaction_vs_fp64_oracle(O, s):
    """the 1-16-16-1 tanh reaction at h = 0.95 beta(s) / rho against the oracle's fp64 RKC2 forward and adjoint, at the bounds
    of test_gpu_parity.test_rkc2_stabilised_solver_fisher_kpp_vs_oracle."""
    nx, N, n_steps = 64, 5, 20
    rng = np.random.default_rng(s)
    D0 = 0.01 * (nx - 1) ** 2
    dt = float(np.float32(0.95 * A.beta(s) / (4 * D0 + 2)))
    theta = np.concatenate([glorot_theta(FK_WIDTHS, seed=3), [1.0, -2.0, 1.0, 0.0, D0]]).astype(np.float32)
    x = np.linspace(0, 1, nx)
    u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / 0.05) - np.tanh((x - (0.5 + d / 2)) / 0.05)) for d in rng.uniform(0.15, 0.5, N)],
                  axis=1).astype(np.float32)
    every = n_steps // 4
    y = (0.9 * np.repeat(u0[None], 5, axis=0)).astype(np.float32)
    sv = fkpp_solver(nx, N, dt, n_steps, every, s)
    sv.set_params(torch.from_numpy(theta).cuda())
    status = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = sv.forward(torch.from_numpy(u0).cuda(), status=status)
    loss, g, gu = sv.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)
    torch.cuda.synchronize()
    out, loss, g, gu, status = out.cpu().numpy(), float(loss), g.cpu().numpy(), gu.cpu().numpy(), status.cpu().numpy()
    sv.close()
    assert (status == 0).all()
    m = O.fkpp_model(nx, FK_WIDTHS, ("tanh", "tanh", "identity"))
    th64 = theta.astype(np.float64)
    l_ref, g_ref, gu_ref, o_ref = 0.0, np.zeros(theta.size), np.zeros((nx, N)), np.zeros((5, nx, N))
    for k in range(N):
        o, us, fs = O.solve_rkc2(m, th64, u0[:, k].astype(np.float64), dt, n_steps, s, save_every=every, want_record=True)
        r = o - y[:, :, k]
        gk, guk = O.adjoint_rkc2(m, th64, us, fs, dt, n_steps, s, 2 * r, save_every=every)
        l_ref += (r ** 2).sum()
        g_ref += gk
        gu_ref[:, k] = guk
        o_ref[:, :, k] = o
    assert np.abs(out - o_ref).max() <= 1e-4 * (1 + np.abs(o_ref).max())
    assert abs(loss - l_ref) <= 1e-3 * abs(l_ref)
    assert np.linalg.norm(g - g_ref) <= 5e-3 * np.linalg.norm(g_ref)
    assert np.abs(gu - gu_ref).max() <= 5e-3 * np.abs(gu_ref).max()
