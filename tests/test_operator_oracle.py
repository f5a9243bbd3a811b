"""The wide-state operator UDE (B200UDE_MODEL_OPERATOR, Climate/NeuralPDE/npde.jl) without a GPU: the fp64 reference
(operator_ref.py) against torch autograd through a pure-torch Tsit5, finite differences, a matrix exponential, the oracle's
neural ODE and its own RKC2 convergence; the npde.jl transcription; and the descriptor validation of b200ude_create."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.linalg
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import operator_ref as R  # noqa: E402


def case(d=5, widths=(5, 4, 3), acts=(1, 1), d2=True, seed=0):
    rng = np.random.default_rng(seed)
    m = widths[-1]
    D1 = rng.normal(scale=0.5, size=(d, m))
    D2 = -np.eye(d) + 0.2 * rng.normal(size=(d, d)) if d2 else None
    model = R.Model(widths, acts, D1, D2)
    return model, rng.normal(scale=0.5, size=model.P), rng.normal(scale=0.5, size=d)


def _torch_loss(model, th, u0, dt, n_steps, cot):
    """sum(cot * out) of a pure-torch fixed-step Tsit5, differentiable in theta and u0."""
    D1 = torch.tensor(model.D1)
    D2 = None if model.D2 is None else torch.tensor(model.D2)
    act = {0: lambda z: z, 1: torch.tanh, 2: lambda z: torch.exp(-z * z)}

    def rhs(u):
        x, o = u, 0
        for a, b, k in zip(model.widths[:-1], model.widths[1:], model.acts):
            W = th[o:o + a * b].reshape(a, b).T
            x = act[k](W @ x + th[o + a * b:o + a * b + b])
            o += a * b + b
        return D1 @ x + (0 if D2 is None else D2 @ u)

    u, k = u0, [None] * 7
    k[0] = rhs(u)
    L = (torch.tensor(cot[0]) * u).sum()
    for s in range(n_steps):
        for i in range(1, 7):
            g = u + dt * sum(float(R.A[i, j]) * k[j] for j in range(i))
            k[i] = rhs(g)
        u = g
        L = L + (torch.tensor(cot[s + 1]) * u).sum()
        k[0] = k[6]
    return L


@pytest.mark.parametrize("acts,d2", [((1, 1), True), ((2, 0), False), ((0, 1), True)])
def test_fixed_grid_reference_matches_torch_autograd_and_finite_differences(acts, d2):
    model, th, u0 = case(acts=acts, d2=d2)
    dt, n = 0.02, 40
    out, rec = R.tsit5_fixed(model, th, u0, 0.0, dt, n)
    cot = np.random.default_rng(1).normal(size=out.shape)
    gth, gu0, _ = R.tsit5_fixed_adjoint(model, th, rec, dt, n, 1, cot)
    tt = torch.tensor(th, requires_grad=True)
    tu = torch.tensor(u0, requires_grad=True)
    _torch_loss(model, tt, tu, dt, n, cot).backward()
    # the interpolating adjoint differs from the discrete gradient by the (4th-order) interpolation error
    assert np.abs(gth - tt.grad.numpy()).max() <= 1e-6 * np.abs(gth).max()
    assert np.abs(gu0 - tu.grad.numpy()).max() <= 1e-6 * np.abs(gu0).max()
    e = 1e-6
    for i in (0, model.P // 2, model.P - 1):
        tp, tm = th.copy(), th.copy()
        tp[i] += e
        tm[i] -= e
        fd = (np.sum(cot * R.tsit5_fixed(model, tp, u0, 0.0, dt, n)[0]) - np.sum(cot * R.tsit5_fixed(model, tm, u0, 0.0, dt, n)[0])) / (2 * e)
        assert abs(fd - gth[i]) <= 1e-6 * max(1.0, abs(fd))


def test_fused_l2_equals_the_explicit_cotangent():
    model, th, u0 = case()
    out, rec = R.tsit5_fixed(model, th, u0, 0.0, 0.05, 20)
    data = out + 0.1
    g1, l1, loss = R.tsit5_fixed_adjoint(model, th, rec, 0.05, 20, 1, data, fused=True)
    g2, l2, _ = R.tsit5_fixed_adjoint(model, th, rec, 0.05, 20, 1, 2 * (out - data))
    np.testing.assert_allclose(g1, g2, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(l1, l2, rtol=1e-12, atol=1e-14)
    assert abs(loss - np.sum((out - data) ** 2)) < 1e-12


def test_adaptive_replay_matches_the_fixed_grid_gradient():
    model, th, u0 = case()
    n_save, save_dt = 11, 0.1
    out, rec, st = R.tsit5_adaptive(model, th, u0, 0.0, save_dt, n_save, 1e-10, 1e-10)
    assert st == 0
    cot = np.random.default_rng(2).normal(size=out.shape)
    g, gu, _ = R.tsit5_adaptive_adjoint(model, th, rec, 0.0, save_dt, n_save, out, cot)
    outf, recf = R.tsit5_fixed(model, th, u0, 0.0, 0.001, 1000, save_every=100)
    gf, guf, _ = R.tsit5_fixed_adjoint(model, th, recf, 0.001, 1000, 100, cot)
    assert np.abs(out - outf).max() < 1e-8
    assert np.abs(g - gf).max() < 1e-6 * np.abs(gf).max() and np.abs(gu - guf).max() < 1e-6 * np.abs(guf).max()


def test_rkc2_adjoint_converges_at_order_two():
    model, th, u0 = case()
    T, ns = 1.0, 10
    cot = np.random.default_rng(3).normal(size=(ns + 1, model.d))
    outf, recf = R.tsit5_fixed(model, th, u0, 0.0, T / 1000, 1000, save_every=100)
    gref, _, _ = R.tsit5_fixed_adjoint(model, th, recf, T / 1000, 1000, 100, cot)
    errs = []
    for n in (20, 40, 80):
        out, rec = R.rkc2_fixed(model, th, u0, T / n, n, 5, save_every=n // ns)
        g, _, _ = R.rkc2_adjoint(model, th, rec, T / n, n, 5, n // ns, cot)
        errs.append(np.abs(g - gref).max())
    r1, r2 = errs[0] / errs[1], errs[1] / errs[2]
    assert 3.2 < r1 < 5.0 and 3.2 < r2 < 5.0, errs


def test_rkc2_reference_matches_the_oracle_on_a_neural_ode():
    from oracle import oracle as O
    model, th, u0 = case(d=3, widths=(3, 8, 3), acts=(1, 0), d2=False)
    model.D1 = np.eye(3)
    m = O.make_model(3, 3, [3, 8, 3], ["tanh", "identity"])   # MODEL_NODE
    out, us, fs = O.solve_rkc2(m, th, u0, 0.05, 20, 4, want_record=True)
    mine, rec = R.rkc2_fixed(model, th, u0, 0.05, 20, 4)
    assert np.abs(mine - out).max() < 1e-12
    cot = np.random.default_rng(4).normal(size=out.shape)
    g, gu = O.adjoint_rkc2(m, th, us, fs, 0.05, 20, 4, cot)
    g2, gu2, _ = R.rkc2_adjoint(model, th, rec, 0.05, 20, 4, 1, cot)
    assert np.abs(g - g2).max() < 1e-11 and np.abs(gu - gu2).max() < 1e-11


@pytest.mark.parametrize("tol", [(1e-6, 1e-3), (1e-8, 1e-8)])
def test_adaptive_reference_matches_the_oracle_neural_ode(tol):
    """With D1 = I and D2 = 0 the adaptive reference is a neural ODE: its saves, accepted-step count and replay gradient agree
    with the oracle's own adaptive Tsit5 (PI controller, initial step, free-interpolant saves) and replay adjoint."""
    from oracle import oracle as O
    model, th, u0 = case(d=4, widths=(4, 16, 4), acts=(1, 0), d2=False, seed=5)
    model.D1 = np.eye(4)
    m = O.make_model(3, 4, [4, 16, 4], ["tanh", "identity"])   # MODEL_NODE
    saveat = np.linspace(0.0, 2.0, 11)
    ref, rec_o = O.solve_adaptive_dense(m, th, u0, saveat, *tol)
    out, rec, st = R.tsit5_adaptive(model, th, u0, 0.0, saveat[1], 11, *tol)
    assert st == 0 and len(rec[0]) == rec_o[3]
    assert np.abs(out - ref).max() < 1e-12
    cot = np.random.default_rng(6).normal(size=out.shape)
    g_o, gu_o = O.adjoint_replay(m, th, saveat, rec_o, cot)
    g, gu, _ = R.tsit5_adaptive_adjoint(model, th, rec, 0.0, saveat[1], 11, out, cot)
    assert np.abs(g - g_o).max() < 1e-11 * max(1.0, np.abs(g_o).max()) and np.abs(gu - gu_o).max() < 1e-11 * max(1.0, np.abs(gu_o).max())


def test_linear_operator_matches_the_matrix_exponential():
    model, th, u0 = case()
    model.D1 = np.zeros_like(model.D1)
    out, _ = R.tsit5_fixed(model, th, u0, 0.0, 0.01, 100, save_every=10)
    for i in range(out.shape[0]):
        np.testing.assert_allclose(out[i], scipy.linalg.expm(model.D2 * 0.1 * i) @ u0, rtol=0, atol=1e-9)


def test_identity_operator_matches_the_oracle_neural_ode():
    from oracle import oracle as O
    model, th, u0 = case(d=4, widths=(4, 16, 4), acts=(1, 0), d2=False)
    model.D1 = np.eye(4)
    m = O.make_model(3, 4, [4, 16, 4], ["tanh", "identity"])   # MODEL_NODE
    ref = O.solve_fixed(m, th, u0, 0.05, 20)
    out, _ = R.tsit5_fixed(model, th, u0, 0.0, 0.05, 20)
    assert np.abs(out - ref).max() < 1e-12


def test_npde_transcription():
    D1, D2 = R.npde_ops()
    assert D1.shape == D2.shape == (30, 30)
    assert abs(np.max(np.abs(np.linalg.eigvals(D2))) - 191.7) < 0.05   # EIGEN_EST of the script
    u0 = R.npde_u0()
    J = D1 @ np.diag(R._dphi(u0)) + D2
    ev = np.linalg.eigvals(J)
    assert abs(np.max(np.abs(ev)) - 218) < 1.0 and abs(np.max(ev.real) + 0.76) < 0.01
    saveat = np.linspace(0, 1.5, 30)
    truth = R.npde_truth(saveat)
    model = R.Model([30, 30], [0], D1, D2)   # ode_i is not a chain; check the truth with a tight fixed-step Tsit5 of ode_i itself
    u, dt = u0.copy(), 1.5 / 29 / 40
    f = lambda v: D1 @ R.npde_phi(v) + D2 @ v   # noqa: E731
    for s in range(29 * 40):
        k = [f(u)]
        for i in range(1, 7):
            k.append(f(u + dt * sum(R.A[i, j] * k[j] for j in range(i))))
        u = u + dt * sum(R.B[j] * k[j] for j in range(6))
    assert model.P == 930 and np.abs(u - truth[-1]).max() < 1e-8


# ---------------------------------------------------------------- descriptor validation (no device needed)
def _desc(dtype=0, widths=(30, 8, 30), acts=(1, 1), **kw):
    from universal_differential_equations_b200 import _lib
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim = dtype, _lib.MODEL_OPERATOR, widths[0]
    d.n_layers = len(acts)
    for i, w in enumerate(widths):
        d.widths[i] = w
    for i, a in enumerate(acts):
        d.acts[i] = a
    d.solver, d.sensealg = _lib.TSIT5, _lib.INTERPOLATING_ADJOINT
    d.t0, d.dt, d.n_steps, d.save_every = 0.0, 0.1, 10, 1
    d.max_trajectories = 8
    d.abstol, d.reltol, d.max_steps = 1e-6, 1e-3, 100
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _create(d):
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.b200ude_create(C.byref(d), C.byref(h))
    if h.value:
        L.b200ude_destroy(h)
    return rc, (L.b200ude_last_error(None) or b"").decode()


@pytest.fixture(scope="module")
def nogpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present (the GPU tests cover creation)")


@pytest.mark.parametrize("dtype", [0, 1])
def test_valid_operator_descriptors_reach_the_device_check(nogpu, dtype):
    from universal_differential_equations_b200 import _lib
    for kw in ({}, dict(adaptive=1), dict(solver=_lib.RKC2, n_stages=5), dict(widths=(1, 1), acts=(0,)),
               dict(widths=(64, 64, 64, 64, 64, 64), acts=(1, 1, 1, 1, 2)), dict(widths=(33, 7, 12), acts=(2, 0)),
               dict(flags=_lib.FLAG_APPROX_TANH)):
        rc, msg = _create(_desc(dtype=dtype, **kw))
        assert rc == _lib.ENODEVICE, (kw, msg)
    d = _desc(dtype=dtype, widths=(16, 8, 4), n_loss_weights=16)
    assert _create(d)[0] == _lib.ENODEVICE


@pytest.mark.parametrize("bad,needle", [
    (dict(state_dim=65, widths=(65, 8, 30)), "state_dim"),
    (dict(state_dim=0), "state_dim"),
    (dict(widths=(30, 65, 30)), "width"),
    (dict(widths=(29, 8, 30), state_dim=30), "widths[0]"),
    (dict(n_consts=1), "n_consts"),
    (dict(n_prefix=1), "n_prefix"),
    (dict(acts=(1, 3)), "activation"),
    (dict(n_loss_weights=3), "n_loss_weights"),
    (dict(n_loss_weights=30), "n_loss_weights"),
    (dict(solver=2, n_stages=1), "n_stages"),
    (dict(solver=2, n_stages=65), "n_stages"),
    (dict(solver=2, n_stages=5, adaptive=1), "RKC2"),
    (dict(adaptive=1, abstol=0.0), "adaptive"),
])
def test_malformed_operator_descriptors_are_einval(bad, needle):
    from universal_differential_equations_b200 import _lib
    rc, msg = _create(_desc(**bad))
    assert rc == _lib.EINVAL and "MODEL_OPERATOR" in msg and needle in msg, msg


@pytest.mark.parametrize("dtype", [0, 1])
@pytest.mark.parametrize("what", ["vern7", "discrete", "vern7_dense", "discrete_dense"])
def test_unbuilt_solvers_on_the_operator_model_are_unsupported(dtype, what):
    from universal_differential_equations_b200 import _lib
    kw = {"vern7": dict(solver=_lib.VERN7), "discrete": dict(sensealg=_lib.DISCRETE_ADJOINT),
          "vern7_dense": dict(solver=_lib.VERN7, flags=_lib.FLAG_VERN7_DENSE),
          "discrete_dense": dict(solver=_lib.VERN7, sensealg=_lib.DISCRETE_ADJOINT, flags=_lib.FLAG_DISCRETE_DENSE, adaptive=1)}[what]
    rc, msg = _create(_desc(dtype=dtype, **kw))
    assert rc == _lib.EUNSUPPORTED and "MODEL_OPERATOR" in msg, msg


def test_python_form_checks_operator_shapes():
    import universal_differential_equations_b200 as ude
    chain = ude.FastChain(ude.FastDense(30, 8, ude.tanh), ude.FastDense(8, 30, ude.tanh))
    D1, D2 = R.npde_ops()
    f = ude.OperatorUDE(chain, D1, D2)
    assert f.state_dim == 30 and f.num_params() == 518 and f.model == 6
    with pytest.raises(ValueError):
        ude.OperatorUDE(chain, D1[:, :8])
    with pytest.raises(ValueError):
        ude.OperatorUDE(chain, D1, D2[:5])
