"""The runtime-shape kernels (k_generic.cu in fp32, k_f64.cu in fp64) at the edges of their envelope (tests/envelope_cases.py), in
every mode they run, against fp64 references; the fp64 kernels against the closed-form linear neural ODE; the fp64 discrete
adjoint against finite differences of the handle's own loss; the constant-bank limit; and interleaved runtime-shape handles.

fp32 tolerances are multiples of the fp32 error budget recorded on the CPU (test_runtime_shape_envelope_oracle.F32_BUDGET).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import discrete_ref as R  # noqa: E402
import envelope_cases as E  # noqa: E402
import linear_node_ref as LN  # noqa: E402
import vern7_dense_ref as V  # noqa: E402
from helpers import glorot_theta  # noqa: E402
from test_runtime_shape_envelope_oracle import F32_BUDGET, GRAD_STEPS, ORDER_STEPS  # noqa: E402


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


MODES = ["tsit5_interp", "tsit5_adaptive", "tsit5_discrete", "vern7_fixed", "vern7_discrete", "vern7_adaptive_discrete",
         "dense_fixed", "dense_adaptive"]
ADAPTIVE = {"tsit5_adaptive", "vern7_adaptive_discrete", "dense_adaptive"}
C_ORACLE = {"tsit5_interp", "tsit5_adaptive", "tsit5_discrete", "vern7_fixed"}   # references in C: ragged N = 129
TOL = {torch.float64: 1e-8, torch.float32: 1e-5}


def _solver(name, mode, N, dtype):
    ude = _ude()
    f = E.ude_form(name)
    sdt, ns = E.grid(name)
    alg = ude.Tsit5() if mode.startswith("tsit5") else ude.Vern7(dense=mode.startswith("dense"))
    sens = ude.ForwardDiffSensitivity() if mode.endswith("discrete") else ude.InterpolatingAdjoint()
    kw = dict(max_trajectories=N, dtype=dtype, alg=alg, sensealg=sens)
    if mode in ADAPTIVE:
        return ude.UDESolver(f, 0.0, sdt, ns - 1, 1, adaptive=True, abstol=TOL[dtype], reltol=TOL[dtype], max_steps=1024, **kw)
    return ude.UDESolver(f, 0.0, sdt / 2, 2 * (ns - 1), 2, **kw)


def _reference(O, name, mode, th, u, tol, y=None, cot=None):
    """fp64 reference -> (states[n_save, d, N], loss or None, grad_theta, grad_u0[d, N]) for the L2 loss on y, or for the
    cotangent cot."""
    m = E.oracle_model(O, name)
    sdt, ns = E.grid(name)
    d, N = u.shape
    ts = sdt * np.arange(ns)
    fixed = (sdt / 2, 2 * (ns - 1))
    if mode in ("tsit5_interp", "vern7_fixed"):
        # the interpolating adjoint of a fixed-step Vern7 handle runs over a Tsit5 re-solve: the oracle's Tsit5 adjoint.  A
        # cotangent c is the L2 cotangent of the targets out - c / 2
        if y is None:
            out_t = O.ensemble_loss_grad(m, th, u, np.zeros((ns, d, N)), np.ones(d), *fixed, save_every=2, want_out=True)[3]
            y_eff = out_t - cot / 2
        else:
            y_eff = y
        L, G, GU, OUT = O.ensemble_loss_grad(m, th, u, y_eff, np.ones(d), *fixed, save_every=2, want_out=True)
        if mode == "vern7_fixed":
            OUT = np.stack([O.solve_fixed(m, th, u[:, k], *fixed, solver=O.VERN7, save_every=2) for k in range(N)], axis=2)
        return OUT, (L if y is not None else None), G, GU
    OUT, G, GU = np.zeros((ns, d, N)), np.zeros(len(th)), np.zeros((d, N))
    for k in range(N):
        def dl(out):
            return 2 * (out - y[:, :, k]) if y is not None else cot[:, :, k]
        if mode == "tsit5_adaptive":
            out, rec = O.solve_adaptive_dense(m, th, u[:, k], ts, tol, tol)
            g, gu = O.adjoint_replay(m, th, ts, rec, dl(out))
        elif mode == "tsit5_discrete":
            out, dense = O.solve_fixed(m, th, u[:, k], *fixed, save_every=2, want_dense=True)
            g, gu = O.adjoint_discrete(m, th, out, dense, *fixed, dl(out), save_every=2)
        elif mode == "vern7_discrete":
            rec = R.fixed_record(fixed[1], fixed[0], 2)
            out, ustep = R.solve_steps(O, m, th, u[:, k], rec, R.VERN7)
            g, gu = R.adjoint_steps(O, m, th, ustep, rec, R.VERN7, dl(out))
        elif mode == "vern7_adaptive_discrete":
            out, rec = R.vern7_adaptive_record(O, m, th, u[:, k], 0.0, sdt, ns, tol, tol)
            g, gu = R.adjoint_steps(O, m, th, rec["ustep"], rec, R.VERN7, dl(out))
        elif mode == "dense_fixed":
            out, rec = V.fixed_record(O, m, th, u[:, k], 0.0, *fixed, 2)
            g, gu = V.replay_adjoint(O, m, th, rec, 0.0, sdt, ns, dl(out))
        else:
            out, rec = V.dense_record(O, m, th, u[:, k], 0.0, sdt, ns, tol, tol)
            g, gu = V.replay_adjoint(O, m, th, rec, 0.0, sdt, ns, dl(out))
        OUT[:, :, k], GU[:, k] = out, gu
        G += g
    return OUT, (float(((OUT - y) ** 2).sum()) if y is not None else None), G, GU


def _run(solver, th, u, y, cot, dtype):
    npd = np.float64 if dtype == torch.float64 else np.float32
    solver.set_params(torch.from_numpy(np.asarray(th, npd)).cuda())
    status = torch.full((u.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(np.asarray(u, npd)).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(np.asarray(y, npd)).cuda(), want_grad_u0=True)
    gc, guc = solver.adjoint(torch.from_numpy(np.asarray(cot, npd)).cuda(), want_grad_u0=True)
    torch.cuda.synchronize()
    return dict(out=out.cpu().numpy().astype(np.float64), loss=float(loss), g=g.cpu().numpy().astype(np.float64),
                gu=gu.cpu().numpy().astype(np.float64), gc=gc.cpu().numpy().astype(np.float64),
                guc=guc.cpu().numpy().astype(np.float64), status=status.cpu().numpy())


def _inputs(O, name, N, dtype):
    th, u = E.theta(name), E.u0(name, N)
    y = E.data(O, name, th, u)
    cot = np.random.default_rng(7).standard_normal(y.shape) * (np.abs(y).max(axis=(0, 2), keepdims=True) + 1)
    if dtype == torch.float32:   # the reference sees the fp32-rounded inputs
        th, u, y, cot = (a.astype(np.float32).astype(np.float64) for a in (th, u, y, cot))
    return th, u, y, cot


def _errors(r, OUT, L, G, GU, Gc, GUc):
    sc = np.abs(OUT).max(axis=(0, 2), keepdims=True) + 1.0
    return dict(states=(np.abs(r["out"] - OUT) / sc).max(), loss=abs(r["loss"] - L) / abs(L),
                grad=np.linalg.norm(r["g"] - G) / np.linalg.norm(G), gu0=np.abs(r["gu"] - GU).max() / np.abs(GU).max(),
                grad_cot=np.linalg.norm(r["gc"] - Gc) / np.linalg.norm(Gc), gu0_cot=np.abs(r["guc"] - GUc).max() / np.abs(GUc).max())


# fp64 against the fp64 references; fixed step: the same arithmetic in another order (round-off); adaptive: the same controller,
# so the same step sequence up to round-off in the accept / reject decisions.  Measured on an H100 (every shape, mode, state /
# loss / gradient / cotangent-gradient error): fixed step <= 1.4e-14, adaptive <= 1.6e-10 (node8_neck, adaptive Tsit5)
F64_BOUND = {"fixed": 1e-12, "adaptive": 2e-9}


def _f32_bound(name, mode, key):
    """K x the CPU fp32 budget (fixed step), plus the solver tolerance's share for the adaptive modes.  The loss is a sum of
    squared residuals of the fp32 states, so its budget is at least the states' one (SEIR: states of 1e4, residuals of 5 %).
    Measured on an H100: every error <= 0.11 of its bound, i.e. <= 11 x budget (SEIR loss 1.0e-6 against a states budget of
    4.3e-7)."""
    s, l, g, gu = F32_BUDGET[name]
    b = dict(states=s, loss=max(l, s), grad=g, gu0=gu, grad_cot=g, gu0_cot=gu)[key]
    K = 100
    if mode in ADAPTIVE:
        return max(K * b, dict(states=50, loss=100, grad=500, gu0=500, grad_cot=500, gu0_cot=500)[key] * TOL[torch.float32])
    return K * b


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", E.F64_SHAPES)
def test_f64_envelope_shape_vs_reference(O, name, mode):
    N = 129 if mode in C_ORACLE else 3
    th, u, y, cot = _inputs(O, name, N, torch.float64)
    solver = _solver(name, mode, N, torch.float64)
    r = _run(solver, th, u, y, cot, torch.float64)
    solver.close()
    tol = TOL[torch.float64]
    OUT, L, G, GU = _reference(O, name, mode, th, u, tol, y=y)
    _, _, Gc, GUc = _reference(O, name, mode, th, u, tol, cot=cot)
    assert (r["status"] == 0).all()
    e = _errors(r, OUT, L, G, GU, Gc, GUc)
    print(f"f64 {name} {mode}: " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    bound = F64_BOUND["adaptive" if mode in ADAPTIVE else "fixed"]
    for k, v in e.items():
        assert v <= bound, (k, v)
    if mode != "vern7_fixed":   # (its fused loss is the one of the Tsit5 re-solve the adjoint runs over)
        l_out = float(((r["out"] - y) ** 2).sum())
        assert abs(r["loss"] - l_out) <= 1e-12 * l_out


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", E.F32_SHAPES)
def test_f32_envelope_shape_vs_f64_reference(O, name, mode):
    N = 129 if mode in C_ORACLE else 3
    th, u, y, cot = _inputs(O, name, N, torch.float32)
    solver = _solver(name, mode, N, torch.float32)
    r = _run(solver, th, u, y, cot, torch.float32)
    solver.close()
    tol = TOL[torch.float32]
    OUT, L, G, GU = _reference(O, name, mode, th, u, tol, y=y)
    _, _, Gc, GUc = _reference(O, name, mode, th, u, tol, cot=cot)
    assert (r["status"] == 0).all()
    e = _errors(r, OUT, L, G, GU, Gc, GUc)
    print(f"f32 {name} {mode}: " + " ".join(f"{k} {v:.2e} ({v / _f32_bound(name, mode, k):.3f} of bound)" for k, v in e.items()))
    for k, v in e.items():
        assert v <= _f32_bound(name, mode, k), (k, v, _f32_bound(name, mode, k))


# ---------------------------------------------------------------------------------------------------- the constant-bank limit
def test_constant_bank_limit_and_the_largest_footprints():
    """fp32 theta lives in the 12 288-float constant bank: P = 12 288 is accepted (lv_bank), P = 12 289 (lv_bank1) and the 13 576 of
    node8_max are refused at create with EUNSUPPORTED; fp64 accepts both.  The adjoints of the largest vectors keep one gradient
    vector per warp in shared memory: 4 x 12 289 floats (196 624 B) and 2 x 13 577 doubles (217 232 B), inside the device's
    opt-in limit (232 448 B on an H100)."""
    ude = _ude()
    from universal_differential_equations_b200 import _lib
    assert E.num_params("lv_bank") == E.F32_BANK and E.num_params("lv_bank1") == E.F32_BANK + 1
    assert E.num_params("node8_max") == 13576
    ok = ude.UDESolver(E.ude_form("lv_bank"), 0.0, 0.05, 20, 2, max_trajectories=4)
    assert ok.P == E.F32_BANK
    ok.close()
    for name in ("lv_bank1", "node8_max"):
        with pytest.raises(_lib.B200UDEError) as ex:
            ude.UDESolver(E.ude_form(name), 0.0, 0.05, 20, 2, max_trajectories=4)
        assert ex.value.code == _lib.EUNSUPPORTED and "constant-bank budget" in str(ex.value)
        s = ude.UDESolver(E.ude_form(name), 0.0, 0.05, 20, 2, max_trajectories=4, dtype=torch.float64)
        assert s.P == E.num_params(name)
        s.close()
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert 4 * 4 * (E.F32_BANK + 1) <= optin and 2 * 8 * (13576 + 1) <= optin


# ---------------------------------------------------------------------------------------------------- closed form, fp64 kernels
LINEAR = ["node1_lin", "node8_lin"]


def _linear_run(name, alg, h, n_steps, save_every, y=None, N=3, adaptive=False, tol=None):
    ude = _ude()
    a = dict(tsit5=ude.Tsit5(), vern7=ude.Vern7(), vern7_dense=ude.Vern7(dense=True))[alg]
    kw = dict(adaptive=True, abstol=tol, reltol=tol, max_steps=4096) if adaptive else {}
    s = ude.UDESolver(E.ude_form(name), 0.0, h, n_steps, save_every, max_trajectories=N, alg=a, dtype=torch.float64, **kw)
    s.set_params(torch.from_numpy(E.theta(name)).cuda())
    u = E.u0(name, N)
    status = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = s.forward(torch.from_numpy(u).cuda(), status=status)
    res = [out.cpu().numpy()]
    if y is not None:
        _, g, gu = s.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)
        res += [g.cpu().numpy(), gu.cpu().numpy()]
    assert (status.cpu().numpy() == 0).all()
    s.close()
    return u, res


@pytest.mark.parametrize("alg", ["tsit5", "vern7"])
@pytest.mark.parametrize("name", LINEAR)
def test_f64_fixed_step_kernels_converge_to_expm_at_their_order(name, alg):
    """Same step sizes and bounds as the oracle's test (test_runtime_shape_envelope_oracle.ORDER_STEPS); the kernels' errors are
    the oracle's to round-off (measured on an H100: Tsit5 5.60 / 5.36 and 5.47 / 5.29, Vern7 6.38 / 6.85 and 7.15 / 7.09 for
    node1_lin and node8_lin)."""
    hs, p, margin = ORDER_STEPS[alg]
    errs = []
    for h in hs:
        u, (out,) = _linear_run(name, alg, h, int(round(1 / h)), 1)
        ex = np.stack([LN.solution(E.theta(name), u[:, k], [1.0])[0] for k in range(u.shape[1])], axis=1)
        errs.append(np.abs(out[-1] - ex).max())
    orders = LN.observed_orders(hs, errs)
    print(f"{name} {alg}: errors {errs} orders {orders}")
    assert min(errs) >= 1e-13 and np.all(np.abs(orders - p) <= margin), orders


@pytest.mark.parametrize("alg", ["tsit5", "vern7", "vern7_dense"])
@pytest.mark.parametrize("name", LINEAR)
def test_f64_adaptive_kernels_land_within_the_tolerance(name, alg):
    """abstol = reltol = 1e-10, saves every 0.1 over (0, 1): the error against expm stays below the tolerance (the oracle's
    adaptive Tsit5 / Vern7 solves measure 5e-12 - 1e-11 and 3e-15 - 5e-15; the kernels on an H100: Tsit5 9.6e-12, Vern7
    6.0e-15, Vern7 dense 5.4e-14)."""
    u, (out,) = _linear_run(name, alg, 0.1, 10, 1, adaptive=True, tol=1e-10)
    ex = np.stack([LN.solution(E.theta(name), u[:, k], 0.1 * np.arange(11)) for k in range(u.shape[1])], axis=2)
    err = np.abs(out - ex).max()
    print(f"{name} adaptive {alg}: {err:.2e}")
    assert err <= 1e-10


@pytest.mark.parametrize("alg", ["tsit5", "vern7_dense"])
@pytest.mark.parametrize("name", LINEAR)
def test_f64_interpolating_adjoint_converges_to_the_exact_gradient(name, alg):
    """The interpolating adjoint over fixed-step Tsit5 (4th-order interpolant: expected order >= 4, asserted >= 3.5) and over the
    Vern7 dense output (expected 7, asserted >= 6) converges to the expm_frechet gradient; step sizes and measured orders as in
    test_runtime_shape_envelope_oracle.GRAD_STEPS; measured on an H100: Tsit5 6.04 / 5.68 and 5.69 / 5.39, Vern7 dense
    6.60 / 6.98 and 7.03 / 7.01 for node1_lin and node8_lin."""
    hs, pmin = GRAD_STEPS[alg]
    sdt, ns, N = 0.5, 5, 3
    d = E.SHAPES[name]["widths"][0]
    y = np.random.default_rng(0).uniform(-1, 1, (ns, d, N))
    th = E.theta(name)
    errs, errs_u = [], []
    for h in hs:
        se = int(round(sdt / h))
        u, (out, g, gu) = _linear_run(name, alg, h, (ns - 1) * se, se, y=y, N=N)
        G, GU = np.zeros(len(th)), np.zeros((d, N))
        for k in range(N):
            _, gk, guk, _ = LN.l2(th, u[:, k], sdt * np.arange(ns), y[:, :, k], np.ones(d))
            G, GU[:, k] = G + gk, guk
        errs.append(np.linalg.norm(g - G) / np.linalg.norm(G))
        errs_u.append(np.abs(gu - GU).max() / np.abs(GU).max())
    orders = LN.observed_orders(hs, errs)
    print(f"{name} {alg}: grad errors {errs} orders {orders}; grad_u0 {errs_u}")
    assert min(errs) >= 1e-13 and np.all(orders >= pmin), orders
    assert errs_u[-1] <= 10 * errs[-1] + 1e-12


# ------------------------------------------------------------------------------------------- finite differences, discrete adjoint
@pytest.mark.parametrize("mode", ["tsit5_discrete", "vern7_discrete"])
@pytest.mark.parametrize("name", E.F64_SHAPES)
def test_f64_discrete_adjoint_matches_finite_differences_of_its_own_loss(O, name, mode):
    """g . v against central differences of the handle's own fp64 loss along six random unit directions: independent of
    discrete_ref.py.  Relative agreement 1e-7 (measured on an H100: <= 3.8e-9, lv_bank1 Vern7)."""
    N = 5
    th, u, y, _ = _inputs(O, name, N, torch.float64)
    solver = _solver(name, mode, N, torch.float64)
    ut, yt = torch.from_numpy(u).cuda(), torch.from_numpy(y).cuda()

    def loss_grad(t):
        solver.set_params(torch.from_numpy(t).cuda())
        solver.forward(ut)
        loss, g, _ = solver.adjoint_l2(yt)
        return float(loss), g.cpu().numpy()

    _, g = loss_grad(th)
    rng = np.random.default_rng(11)
    eps = 1e-5 * max(1.0, np.abs(th).max())
    worst = 0.0
    for _ in range(6):
        v = rng.standard_normal(len(th))
        v /= np.linalg.norm(v)
        fd = (loss_grad(th + eps * v)[0] - loss_grad(th - eps * v)[0]) / (2 * eps)
        rel = abs(fd - g @ v) / max(abs(fd), 1e-3 * np.linalg.norm(g))
        worst = max(worst, rel)
    print(f"{name} {mode}: worst relative FD mismatch {worst:.2e}")
    assert worst <= 1e-7
    solver.close()


# ------------------------------------------------------------------------------------------- interleaved runtime-shape handles
def _fkpp():
    ude = _ude()
    nx, N = 26, 5
    chain = ude.FastChain(ude.FastDense(1, 10, ude.tanh), ude.FastDense(10, 20, ude.tanh), ude.FastDense(20, 10, ude.tanh),
                          ude.FastDense(10, 1))
    f = ude.FisherKPPUDE(chain, nx)
    th = np.concatenate([glorot_theta((1, 10, 20, 10, 1), seed=4), [1.1, -2.3, 0.9, 0.0, 0.01 * (nx - 1) ** 2]]).astype(np.float32)
    x = np.linspace(0, 1, nx)
    rng = np.random.default_rng(3)
    u = np.stack([np.exp(-((x - 0.5) / w) ** 2) for w in rng.uniform(0.1, 0.3, N)], axis=1).astype(np.float32)
    y = (np.repeat(u[None], 6, axis=0) + 0.05 * rng.standard_normal((6, nx, N))).astype(np.float32)
    return (lambda: ude.UDESolver(f, 0.0, 0.1, 5, 1, max_trajectories=N, adaptive=True, max_steps=512)), th, u, y


def _envelope_handle(O, name, N=40):
    th, u, y, _ = _inputs(O, name, N, torch.float32)
    return (lambda: _solver(name, "tsit5_interp", N, torch.float32)), th.astype(np.float32), u.astype(np.float32), y.astype(np.float32)


def test_interleaved_runtime_shape_handles_keep_their_shape_tables(O):
    """The runtime-shape kernels read the chain shape from one constant-bank table (c_gen, sent by upload_gen when the handle
    changes) shared by every runtime-shape handle, the Fisher-KPP ones included.  Forward and adjoint calls of lv_bank, node8_neck
    and an adaptive 1-10-20-10-1 Fisher-KPP handle interleaved on one stream, then one handle destroyed and one of another shape
    created: every output is bitwise the handle's output when it runs alone."""
    specs = {"bank": _envelope_handle(O, "lv_bank"), "neck": _envelope_handle(O, "node8_neck"), "fkpp": _fkpp(),
             "mixed": _envelope_handle(O, "lv_mixed5")}

    def cuda(a):
        return torch.from_numpy(a).cuda()

    alone = {}
    for tag, (make, th, u, y) in specs.items():
        s = make()
        s.set_params(cuda(th))
        out = s.forward(cuda(u))
        loss, g, gu = s.adjoint_l2(cuda(y), want_grad_u0=True)
        alone[tag] = [x.cpu().numpy() for x in (out, loss, g, gu)]
        s.close()
    assert not np.array_equal(alone["bank"][1], alone["mixed"][1])

    h = {tag: specs[tag][0]() for tag in ("bank", "neck", "fkpp")}
    for tag in h:
        h[tag].set_params(cuda(specs[tag][1]))
    outs = {tag: h[tag].forward(cuda(specs[tag][2])) for tag in ("bank", "neck", "fkpp")}
    got = {}
    for tag in ("fkpp", "bank", "neck"):   # adjoints in another order than the forwards
        loss, g, gu = h[tag].adjoint_l2(cuda(specs[tag][3]), want_grad_u0=True)
        got[tag] = [x.cpu().numpy() for x in (outs[tag], loss, g, gu)]
    h["neck"].close()
    h["mixed"] = specs["mixed"][0]()
    h["mixed"].set_params(cuda(specs["mixed"][1]))
    for tag in ("mixed", "bank", "fkpp", "mixed"):
        out = h[tag].forward(cuda(specs[tag][2]))
        loss, g, gu = h[tag].adjoint_l2(cuda(specs[tag][3]), want_grad_u0=True)
        r = [x.cpu().numpy() for x in (out, loss, g, gu)]
        assert all(np.array_equal(a, b) for a, b in zip(r, alone[tag])), tag
    for tag in ("bank", "neck", "fkpp"):
        assert all(np.array_equal(a, b) for a, b in zip(got[tag], alone[tag])), tag
    for tag in ("bank", "fkpp", "mixed"):
        h[tag].close()
