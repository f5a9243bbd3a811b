"""Vern7's lazy 7th-order dense output (B200UDE_FLAG_VERN7_DENSE) without a GPU: the kernels' constants against the doubles the
reference serialized, the order conditions of the continuous extension, the fp64 reference algorithms (tests/vern7_dense_ref.py)
against the reference's stored artefacts, an error-controlled backward solve and finite differences, and the descriptor
validation of the flag."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import vern7_dense_ref as V
from helpers import glorot_theta, theta_scenario1_init

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RBF3 = ("rbf", "rbf", "rbf", "identity")
SEIR_W = np.array([0, 1, 1, 1, 0, 0, 0], np.float64)


def _kernel_constants():
    """The 140 doubles after the tableau (block indices 58..197) as csrc/vern7_dense.cuh spells them, in the block's order."""
    src = open(os.path.join(ROOT, "universal_differential_equations_b200", "csrc", "vern7_dense.cuh")).read()
    body = src[src.index("struct Vern7Dense"):src.index("namespace vern7_dense")]
    fn = {}
    for name in ("c", "a", "r"):
        m = re.search(r"static constexpr double %s\(int i(?:, int [jp])?\)\s*\{(.*?)\n    \}" % name, body, re.S)
        fn[name] = {tuple(int(x) for x in re.findall(r"\d+", key)): float(val)
                    for key, val in re.findall(r"case ([\d *+]+): return ([-+0-9.e]+);", m.group(1))}
    out = []
    for i in range(10, 16):
        out.append(fn["c"][(i,)])
        out += [fn["a"][(i, 16, j)] for j in V._EXTRA_COLS[i]]
    out += [fn["r"][(0, 8, p)] for p in range(1, 8)]
    for i in V.WEIGHTED[1:]:
        out += [fn["r"][(i, 8, p)] for p in range(2, 8)]
    c_update = [fn["c"][(i,)] for i in range(1, 9)]
    return np.array(out), np.array(c_update)


def test_kernel_constants_are_the_serialized_doubles(golden):
    v = golden["scenario_1"]["vern7_consts"]
    assert v.shape == (198,) and v[197] == 0.0
    k, c_update = _kernel_constants()
    assert k.shape == (139,)
    assert np.array_equal(k.view(np.uint64), v[58:197].view(np.uint64))
    assert np.array_equal(c_update[:7].view(np.uint64), v[0:7].view(np.uint64)) and c_update[7] == 1.0
    assert np.array_equal(V.serialized_block(), v)


def test_extra_stage_rows_satisfy_the_simplifying_conditions():
    A, c = V.T["A"], V.T["c"]
    for i in range(10, 16):
        for p in range(4):
            assert abs((A[i] * c**p).sum() - c[i] ** (p + 1) / (p + 1)) <= 1e-16, (i, p)


def test_interpolation_weights_at_theta_one():
    b1 = V.weights(1.0)
    b = V.T["b"]
    for i in V.UPDATE:
        assert abs(b1[i] - b[i]) <= 3e-13, (i, b1[i], b[i])
    for i in range(10, 16):
        assert abs(b1[i]) <= 3e-13, (i, b1[i])   # sums of coefficients up to 1.2e3: round-off
    assert b1[1] == b1[2] == b1[9] == 0.0


@pytest.mark.parametrize("th", [0.2, 0.5, 0.77])
def test_continuous_quadrature_conditions(th):
    bw, c = V.weights(th), V.T["c"]
    for k in range(1, 8):
        assert abs((bw * c ** (k - 1)).sum() - th**k / k) <= 1e-13, (k, th)
    assert abs((bw * c**7).sum() - th**8 / 8) > 1e-6   # a 7th-order extension, not 8th


def test_interpolant_converges_at_seventh_order(O):
    """Fixed-step Vern7 of the NODE du = tanh(W u + b) chain; the interpolant at the step midpoints against a tight solve."""
    from scipy.integrate import solve_ivp
    m = O.make_model(O.MODEL_NODE, 2, (2, 2), ("tanh",))
    th = np.array([0.3, -1.1, 0.9, 0.2, 0.1, -0.2])
    u0 = np.array([0.5, -0.3])
    ref = solve_ivp(lambda t, u: O.rhs(m, th, u), (0, 2), u0, method="DOP853", rtol=1e-14, atol=1e-14, dense_output=True)
    errs = []
    hs = (0.4, 0.2, 0.1)
    for h in hs:
        n = int(round(2 / h))
        _, rec = V.fixed_record(O, m, th, u0, 0.0, h, n, 1)
        e = 0.0
        for s in range(n):
            k = V.stages(O, m, th, rec["ustep"][s], h)
            for th_ in (0.3, 0.5, 0.8):
                e = max(e, np.abs(V.interpolate(rec["ustep"][s], h, k, th_) - ref.sol(s * h + th_ * h)).max())
        errs.append(e)
    orders = np.log2(np.array(errs[:-1]) / np.array(errs[1:]))
    assert orders.min() > 6.5, (errs, orders)


def test_scenario1_stored_solution_by_the_interpolant(O, golden):
    """solve(prob, Vern7(); saveat = 0:0.05:3, abstol = reltol = 1e-6) from the stored start and trained parameters, saves from the
    interpolant (17 steps for 61 save points).  Up to t = 2.85 this is the reference's own computation: the stored X-hat to
    round-off (measured 2.2e-12; with the save times as tstops: 1.3e-7).  The three save points inside the last step differ by
    up to 3.9e-7 (measured); the reference's final step is not the one taken here, and the artefacts do not say why."""
    g = golden["scenario_1"]
    m = O.lv_model((2, 5, 5, 5, 2), RBF3)
    out, rec = V.dense_record(O, m, g["theta_trained"].astype(np.float64), g["X"][:, 0].astype(np.float64), 0.0, 0.05, 61, 1e-6, 1e-6)
    assert len(rec["hstep"]) < 30   # far fewer steps than save points: the saves come from the interpolant
    err = np.abs(out.T - g["Xhat"]).max(axis=0)
    assert err[:58].max() <= 1e-11, err[:58].max()
    assert err.max() <= 5e-7, err.max()


def _lv(O, seed=0):
    m = O.lv_model((2, 5, 5, 5, 2), RBF3, n_prefix=1)
    theta = np.concatenate([[1.7], glorot_theta((2, 5, 5, 5, 2), seed=2).astype(np.float64)])
    u0 = np.array([0.44249296, 4.6280594])
    y = np.random.default_rng(seed).uniform(0.5, 4.0, (31, 2))
    return m, theta, u0, (0.0, 0.1, 31), y, np.ones(2)


def _seir(O, seed=0):
    m = O.seir_model()
    theta = 0.5 * glorot_theta((3, 64, 64, 1), seed=4).astype(np.float64)
    u0 = np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])
    y = O.solve_fixed(m, 0.9 * theta, u0, 0.25, 84, save_every=4) * np.random.default_rng(seed).uniform(0.9, 1.1, (22, 7))
    return m, theta, u0, (0.0, 1.0, 22), y, SEIR_W


@pytest.mark.parametrize("form", ["lv", "seir"])
def test_replay_adjoint_matches_error_controlled_backward_solve(O, form):
    """The replay (the kernels' algorithm) against DiffEqSensitivity's formulation: an error-controlled backward Vern7 solve of
    [lambda; mu] with the save times as tstops and u(t) from the forward's interpolant."""
    m, theta, u0, (t0, sdt, ns), y, w = (_lv if form == "lv" else _seir)(O)
    tol = 1e-6
    out, rec = V.dense_record(O, m, theta, u0, t0, sdt, ns, tol, tol)
    assert len(rec["hstep"]) < ns - 1 or form == "seir"
    cot = 2 * w * (out - y)
    g, gu = V.replay_adjoint(O, m, theta, rec, t0, sdt, ns, cot)
    g2, gu2, nb = V.backward_solve(O, m, theta, rec, t0, sdt, ns, cot, 1e-9, 1e-9)
    assert nb > 0
    # measured 3.3e-11 (LV) and 5.1e-11 (SEIR) relative, grad_theta and grad_u0 alike: both integrate the adjoint of the same
    # interpolated trajectory, one on the forward's steps, the other under error control at 1e-9
    assert np.linalg.norm(g - g2) <= 1e-9 * np.linalg.norm(g2), np.linalg.norm(g - g2) / np.linalg.norm(g2)
    assert np.abs(gu - gu2).max() <= 1e-9 * np.abs(gu2).max()


def test_replay_adjoint_matches_finite_differences_of_the_interpolated_save_loss(O):
    """Central differences of the interpolated-save loss at tolerance 1e-12, where the continuous adjoint and the differences of
    the solve both approach the exact gradient."""
    m, theta, u0, (t0, sdt, ns), y, w = _lv(O)
    tol = 1e-12

    def loss(th, u):
        o, _ = V.dense_record(O, m, th, u, t0, sdt, ns, tol, tol)
        return float((w * (o - y) ** 2).sum())
    out, rec = V.dense_record(O, m, theta, u0, t0, sdt, ns, tol, tol)
    g, gu = V.replay_adjoint(O, m, theta, rec, t0, sdt, ns, 2 * w * (out - y))
    rng = np.random.default_rng(3)
    for _ in range(2):
        v = rng.standard_normal(len(theta))
        v /= np.linalg.norm(v)
        eps = 1e-4
        fd = (loss(theta + eps * v, u0) - loss(theta - eps * v, u0)) / (2 * eps)
        assert abs(fd - g @ v) <= 1e-6 * max(abs(fd), 1e-3 * np.linalg.norm(g)), (fd, g @ v)
    for k in range(m.d):
        e = np.zeros(m.d)
        e[k] = 1e-5
        fd = (loss(theta, u0 + e) - loss(theta, u0 - e)) / (2e-5)
        assert abs(fd - gu[k]) <= 1e-6 * abs(fd) + 1e-8 * np.abs(gu).max(), (k, fd, gu[k])


def test_kat4_adam_replay_with_the_interpolating_adjoint(O, golden):
    """scenario_1.jl:84-87,114 with the interpolating adjoint over the Vern7 dense output instead of ForwardDiffSensitivity: from the
    stored initial parameters through ADAM(0.1), the stored losses[0..5] to 1e-6 relative (measured 3.6e-7; the discrete adjoint
    of the tstops solve is held to 2e-6).  A continuous adjoint agrees with the reference's discrete gradient only to the solver
    tolerance, and the loss itself is now that of the reference's step sequence."""
    g = golden["scenario_1"]
    m = O.lv_model((2, 5, 5, 5, 2), RBF3)
    th = theta_scenario1_init(g)
    X = g["X"].T
    mm, vv = np.zeros_like(th), np.zeros_like(th)
    b1, b2, eta, eps = 0.9, 0.999, 0.1, 1e-8
    worst = 0.0
    for it in range(1, 7):
        out, rec = V.dense_record(O, m, th, X[0], 0.0, 0.1, 31, 1e-6, 1e-6)
        l = ((out - X) ** 2).sum()
        worst = max(worst, abs(l - g["losses"][it - 1]) / g["losses"][it - 1])
        gr, _ = V.replay_adjoint(O, m, th, rec, 0.0, 0.1, 31, 2 * (out - X))
        mm = b1 * mm + (1 - b1) * gr
        vv = b2 * vv + (1 - b2) * gr * gr
        th = th - eta * (mm / (1 - b1**it)) / (np.sqrt(vv / (1 - b2**it)) + eps)
    assert worst <= 1e-6, worst


def _desc(_lib, model, dtype, solver, adaptive, sensealg, flags):
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.solver, d.adaptive, d.sensealg, d.flags = dtype, model, solver, adaptive, sensealg, flags
    if model == _lib.MODEL_LV:
        widths, acts, d.state_dim, d.n_prefix = (2, 5, 5, 5, 2), (2, 2, 2, 0), 2, 1
        d.n_consts = 2; d.consts[0], d.consts[1] = 1.3, 1.8
    elif model in (_lib.MODEL_SEIR, _lib.MODEL_SEIR_NODE):
        widths, acts = ((3, 64, 64, 1), (1, 1, 0)) if model == _lib.MODEL_SEIR else ((7, 16, 7), (1, 0))
        d.state_dim, d.n_consts = 7, 9
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


def test_vern7_dense_descriptors_without_a_gpu():
    """The flag with Vern7 and the interpolating adjoint on the LV / SEIR / SEIR_NODE / NODE forms, fixed and adaptive, fp32 and fp64,
    passes validation (ENODEVICE here); with the discrete adjoint, Tsit5, RKC2 or the Fisher-KPP UPDE it is EUNSUPPORTED."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    F, IA, DA = _lib.FLAG_VERN7_DENSE, _lib.INTERPOLATING_ADJOINT, _lib.DISCRETE_ADJOINT
    for dtype in (_lib.F32, _lib.F64):
        for model in (_lib.MODEL_LV, _lib.MODEL_SEIR, _lib.MODEL_SEIR_NODE, _lib.MODEL_NODE):
            for adaptive in (0, 1):
                rc = L.b200ude_create(C.byref(_desc(_lib, model, dtype, _lib.VERN7, adaptive, IA, F)), C.byref(h))
                assert rc == _lib.ENODEVICE and not h.value, (dtype, model, adaptive, L.b200ude_last_error(None))
        refused = [(_lib.MODEL_LV, _lib.VERN7, 0, DA), (_lib.MODEL_LV, _lib.VERN7, 1, DA), (_lib.MODEL_SEIR, _lib.VERN7, 1, DA),
                   (_lib.MODEL_LV, _lib.TSIT5, 0, IA), (_lib.MODEL_SEIR, _lib.TSIT5, 1, IA), (_lib.MODEL_FKPP, _lib.VERN7, 1, IA),
                   (_lib.MODEL_FKPP, _lib.VERN7, 1, DA), (_lib.MODEL_FKPP, _lib.RKC2, 0, IA)]
        for model, solver, adaptive, sa in refused:
            rc = L.b200ude_create(C.byref(_desc(_lib, model, dtype, solver, adaptive, sa, F)), C.byref(h))
            assert rc == _lib.EUNSUPPORTED, (dtype, model, solver, adaptive, sa)
            assert b"B200UDE_FLAG_VERN7_DENSE" in L.b200ude_last_error(None)
