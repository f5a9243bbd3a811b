"""Discrete adjoint through Vern7's interpolated saves (B200UDE_FLAG_DISCRETE_DENSE) without a GPU: the fp64 reference the kernels
are compared against (tests/vern7_dense_discrete_ref.py), checked against torch autograd through the frozen-step scheme with
interpolated saves, finite differences of that scheme, the tstops discrete adjoint where every save is a step end, and the
reference's stored loss history (KAT-4) on the scripts' own step sequence; and the descriptor validation of the flag."""
import ctypes as C

import numpy as np
import pytest

import discrete_ref as R
import vern7_dense_discrete_ref as DD
import vern7_dense_ref as V
from helpers import glorot_theta, theta_scenario1_init

RBF3 = ("rbf", "rbf", "rbf", "identity")
SEIR_W = np.array([0, 1, 1, 1, 0, 0, 0], np.float64)
FORMS = ["lv0", "lv1", "lv2", "seir", "node"]


def _case(O, form, seed=0):
    """(oracle model, theta, u0, (t0, save_dt, n_save), data, loss weights)."""
    rng = np.random.default_rng(seed)
    if form.startswith("lv"):
        rates = int(form[2])
        acts = ("rbf", "rbf", "tanh", "identity") if rates == 2 else RBF3
        m = O.lv_model((2, 5, 5, 5, 2), acts, n_prefix=rates)
        theta = np.concatenate([[1.3, 1.7][2 - rates:] if rates else [], glorot_theta((2, 5, 5, 5, 2), seed=2)]).astype(np.float64)
        return m, theta, np.array([0.44249296, 4.6280594]), (0.0, 0.1, 31), rng.uniform(0.5, 4.0, (31, 2)), np.ones(2)
    if form == "seir":
        m = O.seir_model()
        theta = 0.5 * glorot_theta((3, 64, 64, 1), seed=4).astype(np.float64)
        u0 = np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])
        y = O.solve_fixed(m, 0.9 * theta, u0, 0.25, 84, save_every=4) * rng.uniform(0.9, 1.1, (22, 7))
        return m, theta, u0, (0.0, 1.0, 22), y, SEIR_W
    m = O.make_model(O.MODEL_NODE, 2, (2, 16, 16, 2), ("tanh", "tanh", "identity"))
    theta = glorot_theta((2, 16, 16, 2), seed=6).astype(np.float64)
    return m, theta, np.array([0.6, -0.4]), (0.0, 0.1, 31), rng.uniform(-1.0, 1.0, (31, 2)), np.ones(2)


@pytest.mark.parametrize("form", FORMS)
def test_adjoint_matches_autograd_through_the_scheme_with_interpolated_saves(O, form):
    torch = pytest.importorskip("torch")
    m, theta, u0, (t0, sdt, ns), y, w = _case(O, form)
    out, rec = V.dense_record(O, m, theta, u0, t0, sdt, ns, 1e-6, 1e-6)
    saves = [s for per in DD.save_map(rec, t0, sdt, ns) for s in per]
    assert sum(th is not None for _, th in saves) >= ns // 2      # most saves come from the interpolant ...
    assert len(rec["hstep"]) < ns - 1 or form == "seir"          # ... because the steps no longer stop at them
    frozen = DD.solve_frozen(O, m, theta, u0, rec, t0, sdt, ns)
    assert np.abs(frozen - out).max() <= 1e-13 * np.abs(out).max()
    g, gu = DD.adjoint_dense_steps(O, m, theta, rec, t0, sdt, ns, 2 * w * (out - y))
    th = torch.tensor(theta, requires_grad=True)
    U0 = torch.tensor(u0, requires_grad=True)
    L = DD.torch_loss(O, m, th, U0, rec, t0, sdt, ns, y, w)
    L.backward()
    assert abs(float(L.detach()) - float((w * (out - y) ** 2).sum())) <= 1e-12 * float(L.detach())
    e_g = np.linalg.norm(g - th.grad.numpy()) / np.linalg.norm(th.grad.numpy())
    e_gu = np.linalg.norm(gu - U0.grad.numpy()) / np.linalg.norm(U0.grad.numpy())
    assert e_g <= 1e-10 and e_gu <= 1e-10, (e_g, e_gu)


@pytest.mark.parametrize("form", ["lv1", "seir"])
def test_adjoint_matches_finite_differences_of_the_frozen_step_solve(O, form):
    m, theta, u0, (t0, sdt, ns), y, w = _case(O, form)
    out, rec = V.dense_record(O, m, theta, u0, t0, sdt, ns, 1e-6, 1e-6)
    g, gu = DD.adjoint_dense_steps(O, m, theta, rec, t0, sdt, ns, 2 * w * (out - y))

    def loss(th, u):
        return float((w * (DD.solve_frozen(O, m, th, u, rec, t0, sdt, ns) - y) ** 2).sum())
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
        assert abs(fd - gu[k]) <= 1e-6 * abs(fd) + 1e-8 * np.abs(gu).max(), (k, fd, gu[k])


@pytest.mark.parametrize("form", ["lv1", "seir"])
def test_equals_the_tstops_discrete_adjoint_when_every_save_is_a_step_end(O, form):
    """On the record of the solve that stops at the save times no save is interpolated and no extra stage enters: the recurrence
    is discrete_ref.adjoint_steps'."""
    m, theta, u0, (t0, sdt, ns), y, w = _case(O, form)
    out, rec = R.vern7_adaptive_record(O, m, theta, u0, t0, sdt, ns, 1e-6, 1e-6)
    assert all(th is None for per in DD.save_map(rec, t0, sdt, ns) for _, th in per)
    cot = 2 * w * (out - y)
    g, gu = DD.adjoint_dense_steps(O, m, theta, rec, t0, sdt, ns, cot)
    g2, gu2 = R.adjoint_steps(O, m, theta, rec["ustep"], rec, R.VERN7, cot)
    assert np.linalg.norm(g - g2) <= 1e-13 * np.linalg.norm(g2)
    assert np.linalg.norm(gu - gu2) <= 1e-13 * np.linalg.norm(gu2)


def test_kat4_adam_replay_on_the_scripts_own_step_sequence(O, golden):
    """scenario_1.jl:84-87,114 as written: Vern7 @ abstol = reltol = 1e-6 stepping freely, saveat = 0.1 from the interpolant,
    ForwardDiffSensitivity, ADAM(0.1), in Float64, from the stored initial parameters.  The loss is that of the reference's step
    sequence (losses[0] to 6e-14).  Measured against the stored history: losses[1..4] within 1.4e-7, losses[5] 3.1e-6 -- further
    than the interpolating adjoint over the same record (3.6e-7) and than the tstops discrete adjoint (6.5e-7).  The gradient here is
    the exact derivative of the 13 frozen steps (autograd agrees to 1e-10, above), so the reference's dual-number solve did not
    differentiate this step sequence; which one it took is not in the stored artefacts.  Held to 1e-6 up to losses[4], 5e-6 at
    losses[5]."""
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
        if it == 6:
            assert worst <= 1e-6, worst
        worst = max(worst, abs(l - g["losses"][it - 1]) / g["losses"][it - 1])
        gr, _ = DD.adjoint_dense_steps(O, m, th, rec, 0.0, 0.1, 31, 2 * (out - X))
        mm = b1 * mm + (1 - b1) * gr
        vv = b2 * vv + (1 - b2) * gr * gr
        th = th - eta * (mm / (1 - b1**it)) / (np.sqrt(vv / (1 - b2**it)) + eps)
    assert worst <= 5e-6, worst


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


def test_discrete_dense_descriptors_without_a_gpu():
    """The flag with Vern7 and the discrete adjoint on the LV / SEIR / SEIR_NODE / NODE forms, fixed and adaptive, fp32 and fp64,
    passes validation (ENODEVICE here); with the interpolating adjoint, Tsit5, RKC2, the Fisher-KPP UPDE or together with
    B200UDE_FLAG_VERN7_DENSE it is EUNSUPPORTED with the flag named; FLAG_VERN7_DENSE with the discrete adjoint stays refused."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    F, FI, IA, DA = _lib.FLAG_DISCRETE_DENSE, _lib.FLAG_VERN7_DENSE, _lib.INTERPOLATING_ADJOINT, _lib.DISCRETE_ADJOINT
    assert F == 4
    for dtype in (_lib.F32, _lib.F64):
        for model in (_lib.MODEL_LV, _lib.MODEL_SEIR, _lib.MODEL_SEIR_NODE, _lib.MODEL_NODE):
            for adaptive in (0, 1):
                rc = L.b200ude_create(C.byref(_desc(_lib, model, dtype, _lib.VERN7, adaptive, DA, F)), C.byref(h))
                assert rc == _lib.ENODEVICE and not h.value, (dtype, model, adaptive, L.b200ude_last_error(None))
        refused = [(_lib.MODEL_LV, _lib.VERN7, 0, IA, F), (_lib.MODEL_LV, _lib.VERN7, 1, IA, F), (_lib.MODEL_SEIR, _lib.VERN7, 1, IA, F),
                   (_lib.MODEL_LV, _lib.TSIT5, 0, DA, F), (_lib.MODEL_SEIR, _lib.TSIT5, 1, DA, F), (_lib.MODEL_NODE, _lib.TSIT5, 1, IA, F),
                   (_lib.MODEL_FKPP, _lib.VERN7, 1, DA, F), (_lib.MODEL_FKPP, _lib.VERN7, 1, IA, F), (_lib.MODEL_FKPP, _lib.RKC2, 0, IA, F),
                   (_lib.MODEL_LV, _lib.VERN7, 1, DA, F | FI), (_lib.MODEL_LV, _lib.VERN7, 1, IA, F | FI)]
        for model, solver, adaptive, sa, flags in refused:
            rc = L.b200ude_create(C.byref(_desc(_lib, model, dtype, solver, adaptive, sa, flags)), C.byref(h))
            assert rc == _lib.EUNSUPPORTED, (dtype, model, solver, adaptive, sa, flags)
            assert b"B200UDE_FLAG_DISCRETE_DENSE" in L.b200ude_last_error(None)
        for adaptive in (0, 1):
            rc = L.b200ude_create(C.byref(_desc(_lib, _lib.MODEL_LV, dtype, _lib.VERN7, adaptive, DA, FI)), C.byref(h))
            assert rc == _lib.EUNSUPPORTED and b"B200UDE_FLAG_VERN7_DENSE" in L.b200ude_last_error(None)
