"""CPU side of the runtime-shape envelope tests.

- The linear neural ODE du/dt = W u + b has closed-form solutions and gradients (tests/linear_node_ref.py: expm and its Frechet
  derivative).  They pin the CPU oracle -- the reference of every GPU solver test -- to something no part of the project wrote:
  fixed-step Tsit5 and Vern7 converge at their orders, adaptive solves land within the tolerance, and the interpolating and
  discrete adjoints converge to the exact continuous gradient.
- The fp32 error budget of every envelope shape (tests/envelope_cases.py): how far the fp32 oracle is from the fp64 oracle.  The
  fp32 GPU tolerances of tests/test_gpu_runtime_shape_envelope.py are multiples of these numbers.
- Shapes outside the envelope are refused at create with EUNSUPPORTED before any device is looked for.
"""
import ctypes as C

import numpy as np
import pytest

import discrete_ref as R
import envelope_cases as E
import linear_node_ref as LN
import vern7_dense_ref as V

LINEAR = ["node1_lin", "node8_lin"]

# fp32 oracle against the fp64 oracle on fp32-rounded inputs (fixed-step Tsit5 + interpolating adjoint, N = 129, the grid of
# envelope_cases.grid), measured on the CPU: relative errors of states (per component, scaled by max |state| + 1), loss,
# |grad_theta| and max |grad_u0|
F32_BUDGET = {
    #              states   loss     grad     grad_u0
    "node1_lin": (8.5e-8, 4.0e-8, 2.6e-7, 1.2e-6),
    "node8_lin": (1.6e-7, 7.7e-8, 4.1e-7, 1.4e-6),
    "node8_neck": (1.3e-7, 9.0e-9, 4.0e-7, 1.8e-6),
    "lv_mixed5": (3.5e-7, 1.3e-7, 3.6e-7, 4.0e-6),
    "lv_bank": (2.6e-7, 1.4e-8, 6.9e-7, 5.1e-6),
    "seir_1L": (4.3e-7, 3.9e-9, 1.8e-8, 4.3e-6),
}


def _case(O, name, N=1):
    m = E.oracle_model(O, name)
    th = E.theta(name)
    u = E.u0(name, N)
    return m, th, u


# ------------------------------------------------------------------------------------------------------------------ closed form
def test_closed_form_helpers_agree_with_each_other():
    """expm of the augmented matrix against the scalar formula; the expm_frechet gradient against central differences of the
    closed-form loss."""
    a, b, u0 = -1.2, 0.7, 0.3
    ts = np.linspace(0.0, 2.0, 9)
    assert np.abs(LN.solution([a, b], [u0], ts)[:, 0] - LN.solution_scalar(a, b, u0, ts)).max() <= 1e-14
    th = E.theta("node8_lin")
    u = E.u0("node8_lin", 1)[:, 0]
    y = np.random.default_rng(0).uniform(-1, 1, (len(ts), 8))
    w = np.linspace(0.5, 1.5, 8)
    L, g, gu, _ = LN.l2(th, u, ts, y, w)
    rng = np.random.default_rng(1)
    for _ in range(3):
        v = rng.standard_normal(len(th))
        eps = 1e-6
        fd = (LN.l2(th + eps * v, u, ts, y, w)[0] - LN.l2(th - eps * v, u, ts, y, w)[0]) / (2 * eps)
        assert abs(fd - g @ v) <= 1e-8 * abs(L), (fd, g @ v)
        vu = rng.standard_normal(8)
        fd = (LN.l2(th, u + eps * vu, ts, y, w)[0] - LN.l2(th, u - eps * vu, ts, y, w)[0]) / (2 * eps)
        assert abs(fd - gu @ vu) <= 1e-8 * abs(L)


# Step sizes with final-time errors between 1e-8 and 1e-12, well above round-off.  Measured orders (successive pairs):
#   node1_lin  Tsit5 h = 0.2, 0.1, 0.05   5.60, 5.36     Vern7 h = 1/2, 1/3, 1/4   6.38, 6.85
#   node8_lin  Tsit5                       5.43, 5.26     Vern7                     7.18, 7.11
ORDER_STEPS = {"tsit5": ([0.2, 0.1, 0.05], 5, 0.6), "vern7": ([0.5, 1 / 3, 0.25], 7, 0.8)}


@pytest.mark.parametrize("alg", ["tsit5", "vern7"])
@pytest.mark.parametrize("name", LINEAR)
def test_oracle_fixed_step_converges_at_its_order(O, name, alg):
    m, th, u = _case(O, name)
    hs, p, margin = ORDER_STEPS[alg]
    ex = LN.solution(th, u[:, 0], [1.0])[0]
    solver = O.TSIT5 if alg == "tsit5" else O.VERN7
    errs = [np.abs(O.solve_fixed(m, th, u[:, 0], h, int(round(1 / h)), solver=solver)[-1] - ex).max() for h in hs]
    orders = LN.observed_orders(hs, errs)
    print(f"{name} {alg}: errors {errs} orders {orders}")
    assert min(errs) >= 1e-13
    assert np.all(np.abs(orders - p) <= margin), orders


@pytest.mark.parametrize("alg", ["tsit5", "vern7"])
@pytest.mark.parametrize("name", LINEAR)
def test_oracle_adaptive_lands_within_the_tolerance(O, name, alg):
    """Measured max error over the save points at abstol = reltol = 1e-10: Tsit5 5.2e-12 / 9.5e-12 (node1_lin /
    node8_lin), Vern7 2.6e-15 / 5.2e-15."""
    m, th, u = _case(O, name)
    ts = np.linspace(0.0, 1.0, 11)
    out, nacc, _ = O.solve_adaptive(m, th, u[:, 0], ts, 1e-10, 1e-10, solver=O.TSIT5 if alg == "tsit5" else O.VERN7)
    err = np.abs(out - LN.solution(th, u[:, 0], ts)).max()
    print(f"{name} adaptive {alg}: {err:.2e} in {nacc} steps")
    assert err <= 1e-10


def _grad_problem(O, name):
    m, th, u = _case(O, name)
    sdt, ns = 0.5, 5
    ts = sdt * np.arange(ns)
    y = np.random.default_rng(0).uniform(-1, 1, (ns, m.d, 1))
    L, G, GU, _ = LN.l2(th, u[:, 0], ts, y[:, :, 0], np.ones(m.d))
    return m, th, u, y, (sdt, ns), L, G, GU


# Interpolating adjoint over fixed-step Tsit5 (backward Tsit5, forward state from the 4th-order free interpolant): expected
# order >= 4; measured 6.1 / 5.7 (node1_lin), 5.8 / 5.4 (node8_lin) at h = 1/2, 1/4, 1/8 over save points 0.5 apart.
# Over Vern7's 7th-order dense output: expected 7; measured 6.7 / 7.0 and 7.1 / 7.0 at h = 1/2, 1/4, 1/6.
GRAD_STEPS = {"tsit5": ([0.5, 0.25, 0.125], 3.5), "vern7_dense": ([0.5, 0.25, 1 / 6], 6.0)}


@pytest.mark.parametrize("alg", ["tsit5", "vern7_dense"])
@pytest.mark.parametrize("name", LINEAR)
def test_oracle_interpolating_adjoint_converges_to_the_exact_gradient(O, name, alg):
    m, th, u, y, (sdt, ns), L, G, GU = _grad_problem(O, name)
    hs, pmin = GRAD_STEPS[alg]
    errs, errs_u = [], []
    for h in hs:
        se = int(round(sdt / h))
        if alg == "tsit5":
            _, g, gu = O.ensemble_loss_grad(m, th, u, y, np.ones(m.d), h, (ns - 1) * se, save_every=se)
            gu = gu[:, 0]
        else:
            out, rec = V.fixed_record(O, m, th, u[:, 0], 0.0, h, (ns - 1) * se, se)
            g, gu = V.replay_adjoint(O, m, th, rec, 0.0, sdt, ns, 2 * (out - y[:, :, 0]))
        errs.append(np.linalg.norm(g - G) / np.linalg.norm(G))
        errs_u.append(np.abs(gu - GU).max() / np.abs(GU).max())
    orders = LN.observed_orders(hs, errs)
    print(f"{name} {alg}: grad errors {errs} orders {orders}; grad_u0 {errs_u}")
    assert min(errs) >= 1e-13 and np.all(orders >= pmin), orders
    assert errs_u[-1] <= 10 * errs[-1] + 1e-12


@pytest.mark.parametrize("alg", ["tsit5", "vern7"])
@pytest.mark.parametrize("name", LINEAR)
def test_discrete_adjoint_references_converge_to_the_exact_gradient(O, name, alg):
    """The discrete adjoint is the exact derivative of the scheme, so it approaches the continuous gradient at the scheme's order:
    the oracle's fixed-step Tsit5 one (O.adjoint_discrete) and discrete_ref's Vern7 one.  Measured orders 5.2 - 6.1 (Tsit5) and
    6.4 - 7.2 (Vern7)."""
    m, th, u, y, (sdt, ns), L, G, GU = _grad_problem(O, name)
    hs, p, margin = ([0.5, 0.25, 0.125], 5, 1.0) if alg == "tsit5" else ([0.5, 0.25, 1 / 6], 7, 1.0)
    errs = []
    for h in hs:
        se = int(round(sdt / h))
        if alg == "tsit5":
            _, g, _ = O.ensemble_loss_grad_discrete(m, th, u, y, np.ones(m.d), h, (ns - 1) * se, save_every=se)
        else:
            rec = R.fixed_record((ns - 1) * se, h, se)
            out, ustep = R.solve_steps(O, m, th, u[:, 0], rec, R.VERN7)
            g, _ = R.adjoint_steps(O, m, th, ustep, rec, R.VERN7, 2 * (out - y[:, :, 0]))
        errs.append(np.linalg.norm(g - G) / np.linalg.norm(G))
    orders = LN.observed_orders(hs, errs)
    print(f"{name} discrete {alg}: grad errors {errs} orders {orders}")
    assert min(errs) >= 1e-13 and np.all(orders >= p - margin), orders


@pytest.mark.parametrize("name", LINEAR)
def test_oracle_ensemble_loss_grad_matches_the_closed_form(O, name):
    """O.ensemble_loss_grad at a fine step (h = 1/40) on an ensemble: loss and gradients equal the closed form to 1e-9."""
    m, th, u = _case(O, name, N=7)
    sdt, ns = 0.25, 5
    ts = sdt * np.arange(ns)
    y = np.random.default_rng(3).uniform(-1, 1, (ns, m.d, 7))
    w = np.linspace(0.5, 1.5, m.d)
    L, G, GU = 0.0, np.zeros(len(th)), np.zeros_like(u)
    for k in range(7):
        l, g, gu, _ = LN.l2(th, u[:, k], ts, y[:, :, k], w)
        L, G, GU[:, k] = L + l, G + g, gu
    l64, g64, gu64, out = O.ensemble_loss_grad(m, th, u, y, w, sdt / 10, 10 * (ns - 1), save_every=10, want_out=True)
    assert abs(l64 - L) <= 1e-10 * abs(L)
    assert np.linalg.norm(g64 - G) <= 1e-9 * np.linalg.norm(G)
    assert np.abs(gu64 - GU).max() <= 1e-9 * np.abs(GU).max()
    if m.d == 1:
        W, b = LN.split(th, 1)
        assert np.abs(out[:, 0, :] - LN.solution_scalar(W[0, 0], b[0], u[0][None, :], ts[:, None])).max() <= 1e-10


# ------------------------------------------------------------------------------------------------------------------ fp32 budget
def f32_budget(O, name, N=129):
    """(states, loss, grad, grad_u0) relative errors of the fp32 oracle against the fp64 oracle on fp32-rounded inputs."""
    m, th, u = _case(O, name, N)
    y = E.data(O, name, th, u)
    sdt, ns = E.grid(name)
    th, u, y = (a.astype(np.float32) for a in (th, u, y))
    w = np.ones(m.d)
    args = (sdt / 2, 2 * (ns - 1))
    l32, g32, gu32, o32 = O.ensemble_loss_grad(m, th, u, y, w.astype(np.float32), *args, save_every=2, want_out=True)
    l64, g64, gu64, o64 = O.ensemble_loss_grad(m, th.astype(np.float64), u.astype(np.float64), y.astype(np.float64), w, *args,
                                               save_every=2, want_out=True)
    sc = np.abs(o64).max(axis=(0, 2), keepdims=True) + 1.0
    return ((np.abs(o32 - o64) / sc).max(), abs(l32 - l64) / abs(l64), np.linalg.norm(g32 - g64) / np.linalg.norm(g64),
            np.abs(gu32 - gu64).max() / np.abs(gu64).max())


@pytest.mark.parametrize("name", E.F32_SHAPES)
def test_f32_error_budget_is_what_is_recorded(O, name):
    """The recorded budget is the measurement (within a factor of 3 either way): the GPU fp32 tolerances scale with it."""
    got = f32_budget(O, name)
    print(name, " ".join(f"{x:.2e}" for x in got))
    for x, rec in zip(got, F32_BUDGET[name]):
        assert rec / 3 <= max(x, 1e-12) <= 3 * rec, (got, F32_BUDGET[name])


# ------------------------------------------------------------------------------------------------------------------ refusals
def _desc(_lib, dtype, model, widths, acts, state_dim, n_prefix=0, consts=()):
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim, d.n_layers = dtype, model, state_dim, len(widths) - 1
    for i, w in enumerate(widths):
        d.widths[i] = w
    for i, a in enumerate(acts):
        d.acts[i] = a
    d.n_prefix, d.n_consts = n_prefix, len(consts)
    for i, c in enumerate(consts):
        d.consts[i] = c
    d.dt, d.n_steps, d.save_every, d.max_trajectories = 0.1, 10, 1, 16
    return d


OUTSIDE = {
    "width65": dict(model="lv", widths=(2, 65, 2), state_dim=2),
    "six_layers": dict(model="lv", widths=(2, 8, 8, 8, 8, 8, 2), state_dim=2),
    "node_d9": dict(model="node", widths=(9, 16, 9), state_dim=9),
}


@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("case", list(OUTSIDE))
def test_outside_the_envelope_is_refused_before_the_device(case, dtype):
    """EUNSUPPORTED from create whether or not a GPU is present: the shape is checked before the device is looked for."""
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    c = OUTSIDE[case]
    lv = c["model"] == "lv"
    acts = [_lib.ACT_TANH] * (len(c["widths"]) - 2) + [_lib.ACT_IDENTITY]
    d = _desc(_lib, _lib.F32 if dtype == "f32" else _lib.F64, _lib.MODEL_LV if lv else _lib.MODEL_NODE, c["widths"], acts,
              c["state_dim"], consts=(1.3, 1.8) if lv else ())
    h = C.c_void_p()
    assert L.b200ude_create(C.byref(d), C.byref(h)) == _lib.EUNSUPPORTED and not h.value
    # the same descriptor brought inside the envelope is not refused for its shape
    inside = dict(width65=(2, 64, 2), six_layers=(2, 8, 8, 8, 8, 2), node_d9=(8, 16, 8))[case]
    d = _desc(_lib, d.dtype, d.model, inside, acts[-(len(inside) - 1):], 2 if lv else 8, consts=(1.3, 1.8) if lv else ())
    assert L.b200ude_create(C.byref(d), C.byref(h)) in (_lib.OK, _lib.ENODEVICE)
    if h.value:
        L.b200ude_destroy(h)
