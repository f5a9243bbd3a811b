"""Discrete adjoint (sensealg = ForwardDiffSensitivity) over recorded Tsit5 / Vern7 step sequences: the fp64 reference the GPU
kernels are compared against (tests/discrete_ref.py), checked against torch autograd through the scheme, finite differences
on the frozen steps, the oracle's fixed-step Tsit5 discrete adjoint and the reference's stored loss history (KAT-4); and the
descriptor validation of the new configurations without a GPU."""
import ctypes as C

import numpy as np
import pytest

import discrete_ref as R
from helpers import glorot_theta, theta_scenario1_init

RBF3 = ("rbf", "rbf", "rbf", "identity")
SEIR_W = np.array([0, 1, 1, 1, 0, 0, 0], np.float64)


def _lv(O, seed=0):
    """LV 2-5-5-5-2 rbf with one trainable rate (scenario_2.jl:79-98), random data on 0:0.1:3."""
    m = O.lv_model((2, 5, 5, 5, 2), RBF3, n_prefix=1)
    theta = np.concatenate([[1.7], glorot_theta((2, 5, 5, 5, 2), seed=2).astype(np.float64)])
    u0 = np.array([0.44249296, 4.6280594])
    y = np.random.default_rng(seed).uniform(0.5, 4.0, (31, 2))
    return m, theta, u0, (0.0, 0.1, 31), y, np.ones(2)


def _seir(O, seed=0):
    """SEIR exposure UDE 3-64-64-1 (seir_exposure.jl:114-130), populations of 1.4e7, loss on E, I, R, days 0:21."""
    m = O.seir_model()
    theta = 0.5 * glorot_theta((3, 64, 64, 1), seed=4).astype(np.float64)
    u0 = np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])
    y = O.solve_fixed(m, 0.9 * theta, u0, 0.25, 84, save_every=4) * np.random.default_rng(seed).uniform(0.9, 1.1, (22, 7))
    return m, theta, u0, (0.0, 1.0, 22), y, SEIR_W


def _record(O, m, theta, u0, grid, stepping):
    t0, sdt, ns = grid
    if stepping == "adaptive":
        out, rec = R.vern7_adaptive_record(O, m, theta, u0, t0, sdt, ns, 1e-6, 1e-6)
        return out, rec, R.VERN7
    solver = R.VERN7 if stepping == "vern7_fixed" else R.TSIT5
    rec = R.fixed_record(2 * (ns - 1), sdt / 2, 2)
    out, _ = R.solve_steps(O, m, theta, u0, rec, solver)
    return out, rec, solver


@pytest.mark.parametrize("stepping", ["adaptive", "vern7_fixed", "tsit5_fixed"])
@pytest.mark.parametrize("form", ["lv", "seir"])
def test_discrete_adjoint_matches_autograd_through_the_scheme(O, form, stepping):
    torch = pytest.importorskip("torch")
    m, theta, u0, grid, y, w = (_lv if form == "lv" else _seir)(O)
    out, rec, solver = _record(O, m, theta, u0, grid, stepping)
    if stepping == "adaptive":
        assert len(rec["hstep"]) > grid[2] - 1   # the controller took steps between the save points
        o_orc, _, _ = O.solve_adaptive(m, theta, u0, grid[0] + grid[1] * np.arange(grid[2]), 1e-6, 1e-6, solver=O.VERN7)
        assert np.all(np.abs(out - o_orc) <= 1e-9 * (np.abs(o_orc).max(axis=0) + 1))   # the oracle's Vern7 controller
    outs, ustep = R.solve_steps(O, m, theta, u0, rec, solver)
    assert np.abs(outs - out).max() <= 1e-12 * np.abs(out).max()
    g, gu = R.adjoint_steps(O, m, theta, ustep, rec, solver, 2 * w * (out - y))
    th = torch.tensor(theta, requires_grad=True)
    U0 = torch.tensor(u0, requires_grad=True)
    L = R.torch_loss(O, m, th, U0, rec, solver, y, w)
    L.backward()
    assert abs(float(L.detach()) - float((w * (out - y) ** 2).sum())) <= 1e-12 * float(L.detach())
    assert np.linalg.norm(g - th.grad.numpy()) <= 1e-11 * np.linalg.norm(th.grad.numpy())
    assert np.linalg.norm(gu - U0.grad.numpy()) <= 1e-11 * np.linalg.norm(U0.grad.numpy())
    if stepping == "tsit5_fixed":   # the oracle's own fixed-step Tsit5 discrete adjoint is the same quantity
        n_steps, dt = len(rec["hstep"]), rec["hstep"][0]
        o2, dense = O.solve_fixed(m, theta, u0, dt, n_steps, save_every=2, want_dense=True)
        g2, gu2 = O.adjoint_discrete(m, theta, o2, dense, dt, n_steps, 2 * w * (o2 - y), save_every=2)
        assert np.linalg.norm(g - g2) <= 1e-11 * np.linalg.norm(g2)
        assert np.linalg.norm(gu - gu2) <= 1e-11 * np.linalg.norm(gu2)


@pytest.mark.parametrize("form", ["lv", "seir"])
def test_discrete_adjoint_matches_finite_differences_on_the_frozen_steps(O, form):
    m, theta, u0, grid, y, w = (_lv if form == "lv" else _seir)(O)
    out, rec, solver = _record(O, m, theta, u0, grid, "adaptive")
    _, ustep = R.solve_steps(O, m, theta, u0, rec, solver)
    g, gu = R.adjoint_steps(O, m, theta, ustep, rec, solver, 2 * w * (out - y))

    def loss(th, u):
        o, _ = R.solve_steps(O, m, th, u, rec, solver)
        return float((w * (o - y) ** 2).sum())
    rng = np.random.default_rng(5)
    for _ in range(2):
        v = rng.standard_normal(len(theta))
        v /= np.linalg.norm(v)
        eps = 1e-4
        fd = (loss(theta + eps * v, u0) - loss(theta - eps * v, u0)) / (2 * eps)
        assert abs(fd - g @ v) <= 1e-6 * max(abs(fd), 1e-3 * np.linalg.norm(g)), (fd, g @ v)
    for k in range(m.d):
        if gu[k] == 0.0:
            continue
        e = np.zeros(m.d)
        e[k] = 1e-5 * max(1.0, abs(u0[k]))
        fd = (loss(theta, u0 + e) - loss(theta, u0 - e)) / (2 * e[k])
        # components far below the largest carry the difference's round-off (SEIR: D at 1e-10 next to E, I, R at 1e1)
        assert abs(fd - gu[k]) <= 1e-6 * abs(fd) + 1e-8 * np.abs(gu).max(), (k, fd, gu[k])


def test_kat4_adam_replay_with_the_scripts_own_scheme(O, golden):
    """scenario_1.jl:84-87,114 as written: Vern7 @ abstol = reltol = 1e-6, saveat = 0.1, ForwardDiffSensitivity, ADAM(0.1),
    in Float64.  The discrete gradient of that solve, replayed through ADAM from the stored initial parameters, reproduces the
    stored losses[0..5]."""
    g = golden["scenario_1"]
    m = O.lv_model((2, 5, 5, 5, 2), RBF3)
    th = theta_scenario1_init(g)
    X = g["X"].T
    mm, vv = np.zeros_like(th), np.zeros_like(th)
    b1, b2, eta, eps = 0.9, 0.999, 0.1, 1e-8
    for it in range(1, 7):
        out, rec = R.vern7_adaptive_record(O, m, th, X[0], 0.0, 0.1, 31, 1e-6, 1e-6)
        l = ((out - X) ** 2).sum()
        assert abs(l - g["losses"][it - 1]) <= 2e-6 * g["losses"][it - 1], (it, l, g["losses"][it - 1])
        gr, _ = R.adjoint_steps(O, m, th, rec["ustep"], rec, R.VERN7, 2 * (out - X))
        mm = b1 * mm + (1 - b1) * gr
        vv = b2 * vv + (1 - b2) * gr * gr
        th = th - eta * (mm / (1 - b1**it)) / (np.sqrt(vv / (1 - b2**it)) + eps)


def _desc(_lib, model, dtype, solver, adaptive, sensealg):
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.solver, d.adaptive, d.sensealg = dtype, model, solver, adaptive, sensealg
    if model == _lib.MODEL_LV:
        widths, acts, d.state_dim, d.n_prefix = (2, 5, 5, 5, 2), (2, 2, 2, 0), 2, 1
        d.n_consts = 2; d.consts[0], d.consts[1] = 1.3, 1.8
    elif model == _lib.MODEL_SEIR:
        widths, acts, d.state_dim = (3, 64, 64, 1), (1, 1, 0), 7
        d.n_consts = 9
        for i, c in enumerate((10.0, 0.5944, 0.4239, 1117.3, 0.02, 1 / 3, 1 / 5, 0.2, 1 / 11.2)):
            d.consts[i] = c
    elif model == _lib.MODEL_NODE:
        widths, acts, d.state_dim = (3, 16, 3), (1, 0), 3
    else:   # Fisher-KPP
        widths, acts, d.state_dim, d.n_suffix = (1, 10, 1), (1, 0), 26, 5
    d.n_layers = len(widths) - 1
    for i, x in enumerate(widths):
        d.widths[i] = x
    for i, a in enumerate(acts):
        d.acts[i] = a
    d.dt, d.n_steps, d.save_every, d.max_trajectories = 0.1, 30, 1, 8
    d.abstol, d.reltol, d.max_steps = 1e-6, 1e-6, 512
    if solver == _lib.RKC2:
        d.n_stages = 8
    return d


def test_discrete_adjoint_descriptors_without_a_gpu():
    """Discrete + Vern7 (fixed and adaptive) and discrete + fixed-step Tsit5 on the LV / SEIR / NODE forms, fp32 and fp64, pass
    validation (ENODEVICE here); discrete + adaptive Tsit5, Fisher-KPP and RKC2 are EUNSUPPORTED with a message naming what is
    supported."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    D = _lib.DISCRETE_ADJOINT
    for dtype in (_lib.F32, _lib.F64):
        for model in (_lib.MODEL_LV, _lib.MODEL_SEIR, _lib.MODEL_NODE):
            for solver, adaptive in ((_lib.VERN7, 0), (_lib.VERN7, 1), (_lib.TSIT5, 0)):
                rc = L.b200ude_create(C.byref(_desc(_lib, model, dtype, solver, adaptive, D)), C.byref(h))
                assert rc == _lib.ENODEVICE and not h.value, (dtype, model, solver, adaptive, L.b200ude_last_error(None))
        refused = [(_lib.MODEL_LV, _lib.TSIT5, 1), (_lib.MODEL_SEIR, _lib.TSIT5, 1), (_lib.MODEL_FKPP, _lib.TSIT5, 0),
                   (_lib.MODEL_FKPP, _lib.VERN7, 0), (_lib.MODEL_FKPP, _lib.TSIT5, 1), (_lib.MODEL_FKPP, _lib.RKC2, 0)]
        for model, solver, adaptive in refused:
            rc = L.b200ude_create(C.byref(_desc(_lib, model, dtype, solver, adaptive, D)), C.byref(h))
            assert rc == _lib.EUNSUPPORTED, (dtype, model, solver, adaptive)
            msg = L.b200ude_last_error(None)
            assert b"fixed-step Tsit5" in msg and b"adaptive Vern7" in msg, msg
