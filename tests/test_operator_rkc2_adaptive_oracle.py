"""Adaptive RKC2 on the operator UDE without a GPU: the fp64 reference (operator_rkc2_adaptive_ref.py) against its own step
rule, the fixed-step RKC2 reference, a matrix exponential and its Frechet derivative, adaptive Tsit5, finite differences and
torch autograd; the npde.jl step and right-hand-side counts; and the descriptor validation of b200ude_create."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.linalg
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import operator_ref as R  # noqa: E402
import operator_rkc2_adaptive_ref as A  # noqa: E402


def case(d=5, widths=(5, 4, 3), acts=(1, 1), seed=0, stiff=40.0):
    rng = np.random.default_rng(seed)
    m = widths[-1]
    D1 = rng.normal(scale=0.5, size=(d, m))
    D2 = -stiff * np.eye(d) + 0.2 * rng.normal(size=(d, d))
    model = R.Model(widths, acts, D1, D2)
    return model, rng.normal(scale=0.5, size=model.P), rng.normal(scale=0.5, size=d)


def rho_of(model):
    return float(np.max(np.abs(np.linalg.eigvals(model.D2)))) * 1.2 + 2.0


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def test_beta_matches_the_python_mirror():
    from universal_differential_equations_b200 import sciml
    for s in range(2, 65):
        assert A.beta(s) == sciml._rkc2_beta(s)
        assert A.beta(s) > A.beta(s - 1) if s > 2 else True
    assert 0.6 * 64 ** 2 < A.beta(64) < 0.66 * 64 ** 2


@pytest.mark.parametrize("cap", [64, 4])
def test_step_rule_fewest_stable_stages_and_the_cap(cap):
    model, th, u0 = case(stiff=200.0)
    rho = rho_of(model)
    out, (us, fs, tg, ss), st = A.rkc2_adaptive(model, th, u0, 0.0, 0.5, 5, 1e-4, 1e-2, rho, cap=cap)
    assert st == 0 and np.isfinite(out).all()
    hs = np.diff(tg)
    assert len(ss) == len(hs) > 3
    for h, s in zip(hs, ss):
        assert 2 <= s <= cap
        assert A.beta(s) >= 1.05 * h * rho * (1 - 1e-12)
        if s > 2:   # the fewest such stages, unless the cap cut h
            assert A.beta(s - 1) < 1.05 * h * rho or s == cap
    hcap = A.beta(cap) / (1.05 * rho)
    assert hs.max() <= hcap * (1 + 1e-12)
    if cap == 4:   # the cap binds: steps at exactly beta(cap) / (1.05 rho)
        assert np.sum(np.abs(hs - hcap) <= 1e-12 * hcap) >= len(hs) // 2 and max(ss) == cap
    else:
        assert max(ss) > 4


def test_replay_adjoint_on_a_uniform_record_equals_the_fixed_rkc2_adjoint():
    model, th, u0 = case()
    dt, n, S, every = 0.01, 20, 7, 4
    out, rec = R.rkc2_fixed(model, th, u0, dt, n, S, every)
    cot = np.random.default_rng(3).normal(size=out.shape)
    g_fix, u_fix, _ = R.rkc2_adjoint(model, th, rec, dt, n, S, every, cot)
    arec = (rec[0], rec[1], dt * np.arange(n + 1), [S] * n)
    g_ad, u_ad, _ = A.rkc2_adaptive_adjoint(model, th, arec, 0.0, dt * every, n // every + 1, out, cot)
    assert rel(g_ad, g_fix) < 1e-12 and rel(u_ad, u_fix) < 1e-12
    data = np.random.default_rng(4).normal(size=out.shape)
    g_fix, u_fix, l_fix = R.rkc2_adjoint(model, th, rec, dt, n, S, every, data, fused=True)
    g_ad, u_ad, l_ad = A.rkc2_adaptive_adjoint(model, th, arec, 0.0, dt * every, n // every + 1, out, data, fused=True)
    assert rel(g_ad, g_fix) < 1e-12 and rel(u_ad, u_fix) < 1e-12 and abs(l_ad - l_fix) < 1e-12 * l_fix


def _linear_exact(model, th, u0, ts, cot):
    """saves and (grad_theta, grad_u0) of L = sum_i cot_i . u(t_i) for the one-layer identity chain, from expm and expm_frechet of
    the augmented matrix [[D1 W + D2, D1 b], [0, 0]] acting on [u; 1]."""
    d = model.d
    (W, b, _, _), = model.layers(th)
    M = np.zeros((d + 1, d + 1))
    M[:d, :d] = model.D1 @ W + model.D2
    M[:d, d] = model.D1 @ b
    z0 = np.append(u0, 1.0)
    outs, G, gu = [], np.zeros_like(M), np.zeros(d)
    for t, c in zip(ts, cot):
        E = scipy.linalg.expm(M * t)
        outs.append((E @ z0)[:d])
        ca = np.append(c, 0.0)
        G += t * scipy.linalg.expm_frechet(M.T * t, np.outer(ca, z0), compute_expm=False)
        gu += (E.T @ ca)[:d]
    GW = model.D1.T @ G[:d, :d]   # dL/dW [m, d]
    gb = model.D1.T @ G[:d, d]
    return np.array(outs), np.concatenate([GW.T.ravel(), gb]), gu


def test_linear_chain_converges_to_expm_and_its_frechet_derivative():
    d = 4
    rng = np.random.default_rng(5)
    model = R.Model((d, d), (0,), rng.normal(scale=0.5, size=(d, d)), -30.0 * np.eye(d) + rng.normal(size=(d, d)))
    th = rng.normal(scale=0.5, size=model.P)
    u0 = rng.normal(size=d)
    n_save, save_dt = 6, 0.2
    ts = save_dt * np.arange(n_save)
    cot = rng.normal(size=(n_save, d))
    oref, gref, uref = _linear_exact(model, th, u0, ts, cot)
    rho = float(np.max(np.abs(np.linalg.eigvals(model.D1 @ model.layers(th)[0][0] + model.D2)))) * 1.1
    errs = []
    for tol in (1e-4, 1e-6, 1e-8):
        out, rec, st = A.rkc2_adaptive(model, th, u0, 0.0, save_dt, n_save, tol, tol, rho)
        g, gu, _ = A.rkc2_adaptive_adjoint(model, th, rec, 0.0, save_dt, n_save, out, cot)
        assert st == 0
        errs.append((rel(out, oref), rel(g, gref), rel(gu, uref)))
    print("MEASURED linear chain (forward, grad theta, grad u0) errors at tol 1e-4, 1e-6, 1e-8:", [tuple(f"{x:.1e}" for x in e) for e in errs])
    for k in range(3):
        assert errs[2][k] < errs[1][k] < errs[0][k]
    assert errs[2][0] < 1e-6 and errs[2][1] < 1e-5 and errs[2][2] < 1e-5


def test_gradient_at_tight_tolerance_agrees_with_adaptive_tsit5():
    model, th, u0 = case(stiff=10.0)
    rho = rho_of(model)
    n_save, save_dt = 4, 0.1
    cot = np.random.default_rng(6).normal(size=(n_save, model.d))
    out, rec, st = A.rkc2_adaptive(model, th, u0, 0.0, save_dt, n_save, 1e-9, 1e-9, rho)
    g, gu, _ = A.rkc2_adaptive_adjoint(model, th, rec, 0.0, save_dt, n_save, out, cot)
    o5, rec5, st5 = R.tsit5_adaptive(model, th, u0, 0.0, save_dt, n_save, 1e-12, 1e-12)
    g5, gu5, _ = R.tsit5_adaptive_adjoint(model, th, rec5, 0.0, save_dt, n_save, o5, cot)
    assert st == st5 == 0
    print(f"MEASURED RKC2 at 1e-9 vs Tsit5 at 1e-12: states {rel(out, o5):.1e}, grad theta {rel(g, g5):.1e}, grad u0 {rel(gu, gu5):.1e}")
    assert rel(out, o5) < 1e-6 and rel(g, g5) < 2e-6 and rel(gu, gu5) < 2e-6


def _loss(model, th, u0, data, tol, rho):
    out, _, _ = A.rkc2_adaptive(model, th, u0, 0.0, 0.1, 4, tol, tol, rho)
    return float(np.sum((out - data) ** 2))


def test_gradient_against_finite_differences():
    model, th, u0 = case(stiff=10.0)
    rho, tol = rho_of(model), 1e-9
    data = np.random.default_rng(7).normal(scale=0.3, size=(4, model.d))
    out, rec, _ = A.rkc2_adaptive(model, th, u0, 0.0, 0.1, 4, tol, tol, rho)
    g, gu, l = A.rkc2_adaptive_adjoint(model, th, rec, 0.0, 0.1, 4, out, data, fused=True)
    assert abs(l - _loss(model, th, u0, data, tol, rho)) < 1e-12 * l
    eps = 1e-5
    for k in (0, 7, model.P - 1):
        e = np.zeros(model.P)
        e[k] = eps
        fd = (_loss(model, th + e, u0, data, tol, rho) - _loss(model, th - e, u0, data, tol, rho)) / (2 * eps)
        assert abs(fd - g[k]) < 1e-5 * np.abs(g).max() + 1e-6 * abs(fd), (k, fd, g[k])
    for k in range(model.d):
        e = np.zeros(model.d)
        e[k] = eps
        fd = (_loss(model, th, u0 + e, data, tol, rho) - _loss(model, th, u0 - e, data, tol, rho)) / (2 * eps)
        assert abs(fd - gu[k]) < 1e-5 * np.abs(gu).max(), (k, fd, gu[k])


def test_gradient_against_torch_autograd_through_the_frozen_steps():
    """The replay adjoint is the continuous adjoint discretised on the accepted steps; torch differentiates the forward scheme
    with those steps and stage counts frozen.  The two agree to the solve's accuracy."""
    model, th, u0 = case(stiff=10.0)
    rho, n_save, save_dt = rho_of(model), 4, 0.1
    cot = np.random.default_rng(8).normal(size=(n_save, model.d))
    out, rec, _ = A.rkc2_adaptive(model, th, u0, 0.0, save_dt, n_save, 1e-9, 1e-9, rho)
    g, gu, _ = A.rkc2_adaptive_adjoint(model, th, rec, 0.0, save_dt, n_save, out, cot)
    _, _, tg, ss = rec
    D1, D2 = torch.tensor(model.D1), torch.tensor(model.D2)

    def rhs(tt, u):
        x, o = u, 0
        for a, b in zip(model.widths[:-1], model.widths[1:]):
            x = torch.tanh(tt[o:o + a * b].reshape(a, b).T @ x + tt[o + a * b:o + a * b + b])
            o += a * b + b
        return D1 @ x + D2 @ u

    tt = torch.tensor(th, requires_grad=True)
    ut = torch.tensor(u0, requires_grad=True)
    u, F0 = ut, rhs(tt, ut)
    L, isave = (torch.tensor(cot[0]) * ut).sum(), 1
    for n, s in enumerate(ss):
        h = tg[n + 1] - tg[n]
        tb = A.tables(s)
        Y0, Y1 = u, u + tb["mt1"] * h * F0
        for j in range(2, s + 1):
            F = rhs(tt, Y1)
            Y0, Y1 = Y1, (1 - tb["mu"][j] - tb["nu"][j]) * u + tb["mu"][j] * Y1 + tb["nu"][j] * Y0 + tb["mt"][j] * h * F + tb["ga"][j] * h * F0
        F1 = rhs(tt, Y1)
        while isave < n_save and save_dt * isave <= tg[n + 1] + 1e-12:
            L = L + (torch.tensor(cot[isave]) * A.herm(min((save_dt * isave - tg[n]) / h, 1.0), h, u, Y1, F0, F1)).sum()
            isave += 1
        u, F0 = Y1, F1
    L.backward()
    assert rel(g, tt.grad.numpy()) < 1e-5 and rel(gu, ut.grad.numpy()) < 1e-5


def test_status_words():
    model, th, u0 = case()
    rho = rho_of(model)
    out, rec, st = A.rkc2_adaptive(model, th, u0, 0.0, 0.1, 11, 1e-10, 1e-10, rho, max_steps=5)
    assert st == 2 and len(rec[3]) == 5 and np.isnan(out[-1]).all()
    out, rec, st = A.rkc2_adaptive(model, th, np.full(model.d, np.nan), 0.0, 0.1, 11, 1e-6, 1e-3, rho)
    assert st == 1


@pytest.mark.parametrize("tol,t1,n_save", [((1e-6, 1e-3), 1.5, 30), ((1e-4, 1e-2), 10.0, 195)])
def test_npde_counts_next_to_adaptive_tsit5(tol, t1, n_save):
    """npde.jl's 30-8-30 closure at Glorot theta over its two solves: the training loss at the default tolerances and the t = 10
    solve at (1e-4, 1e-2), adaptive RKC2 with eigen_est = rho(D2) = 191.7 next to adaptive Tsit5."""
    D1, D2 = R.npde_ops()
    model = R.Model([30, 8, 30], [1, 1], D1, D2)
    th = R.glorot([30, 8, 30], np.random.default_rng(0))
    u0 = R.npde_u0()
    save_dt = t1 / (n_save - 1)
    c = {}
    out, rec, st = A.rkc2_adaptive(model, th, u0, 0.0, save_dt, n_save, tol[0], tol[1], 191.7, counts=c)
    o5, rec5, st5 = R.tsit5_adaptive(model, th, u0, 0.0, save_dt, n_save, tol[0], tol[1])
    n5 = len(rec5[0])
    print(f"MEASURED npde {tol} to t = {t1}: adaptive RKC2 {c['accepted']} accepted / {c['rejected']} rejected steps, {c['rhs']} RHS, "
          f"stages {min(rec[3])}..{max(rec[3])}; adaptive Tsit5 {n5} accepted steps; |RKC2 - Tsit5| at t1 {np.abs(out[-1] - o5[-1]).max():.1e}")
    assert st == st5 == 0 and np.isfinite(out).all()
    assert np.abs(out[-1] - o5[-1]).max() < 50 * tol[1]
    assert c["rhs"] < 6 * n5   # Tsit5 spends 6 right-hand sides per accepted step


# ---------------------------------------------------------------- descriptor validation (no device needed)
def _desc(**kw):
    import test_operator_oracle as T
    return T._desc(**kw)


def _create(d):
    import test_operator_oracle as T
    return T._create(d)


@pytest.fixture(scope="module")
def nogpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present (the GPU tests cover creation)")


def _ark(**kw):
    from universal_differential_equations_b200 import _lib
    d = _desc(**{**dict(solver=_lib.RKC2, n_stages=64, adaptive=1, n_consts=1), **kw})
    d.consts[0] = 191.7
    return d


@pytest.mark.parametrize("dtype", [0, 1])
def test_valid_adaptive_rkc2_descriptors_reach_the_device_check(nogpu, dtype):
    from universal_differential_equations_b200 import _lib
    for kw in ({}, dict(n_stages=2), dict(widths=(64, 64, 64), acts=(1, 0)), dict(widths=(1, 4, 1), acts=(1, 0))):
        d = _ark(dtype=dtype, **kw)
        if "widths" in kw:
            d.state_dim = kw["widths"][0]
        rc, msg = _create(d)
        assert rc == _lib.ENODEVICE, (kw, msg)


@pytest.mark.parametrize("rho", [0.0, -1.0, float("nan"), float("inf")])
def test_bad_eigen_est_is_einval(rho):
    from universal_differential_equations_b200 import _lib
    d = _ark()
    d.consts[0] = rho
    rc, msg = _create(d)
    assert rc == _lib.EINVAL and "MODEL_OPERATOR" in msg and "eigen_est" in msg, msg


def test_other_adaptive_rkc2_refusals():
    from universal_differential_equations_b200 import _lib
    rc, msg = _create(_desc(solver=_lib.RKC2, n_stages=64, adaptive=1))   # no eigen_est
    assert rc == _lib.EINVAL and "RKC2" in msg and "eigen_est" in msg and "consts[0]" in msg and "MODEL_OPERATOR" in msg, msg
    rc, msg = _create(_ark(n_consts=2))
    assert rc == _lib.EINVAL and "n_consts" in msg, msg
    rc, msg = _create(_ark(n_stages=65))
    assert rc == _lib.EINVAL and "n_stages" in msg, msg
    d = _desc(solver=_lib.RKC2, n_stages=5, n_consts=1)   # fixed-step RKC2 takes no constant
    d.consts[0] = 191.7
    rc, msg = _create(d)
    assert rc == _lib.EINVAL and "n_consts" in msg, msg
    rc, msg = _create(_ark(sensealg=_lib.DISCRETE_ADJOINT))
    assert rc == _lib.EUNSUPPORTED and "MODEL_OPERATOR" in msg, msg


def test_adaptive_rkc2_on_fisher_kpp_stays_unsupported():
    from universal_differential_equations_b200 import _lib
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim, d.n_layers = 0, _lib.MODEL_FKPP, 16, 3
    for i, w in enumerate((1, 16, 16, 1)):
        d.widths[i] = w
    for i, a in enumerate((1, 1, 0)):
        d.acts[i] = a
    d.n_suffix = 5
    d.n_consts = 1
    d.consts[0] = 191.7
    d.solver, d.n_stages, d.adaptive = _lib.RKC2, 64, 1
    d.t0, d.dt, d.n_steps, d.save_every, d.max_trajectories = 0.0, 0.1, 10, 1, 4
    d.abstol, d.reltol, d.max_steps = 1e-6, 1e-3, 100
    rc, msg = _create(d)
    assert rc == _lib.EUNSUPPORTED, msg
