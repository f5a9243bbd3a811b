"""The discrete adjoint through Vern7's interpolated saves (B200UDE_FLAG_DISCRETE_DENSE, `Vern7(dense=True)` with
`ForwardDiffSensitivity()`) on the GPU, fp64 and fp32: against the fp64 reference (tests/vern7_dense_discrete_ref.py, pinned on
the CPU to autograd through the scheme), the forward against the dense-output handle's, fused against unfused, trajectory
isolation and determinism, a solve that runs out of steps, the fixed-grid convention, and scenario 1's call as written."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import vern7_dense_discrete_ref as DD  # noqa: E402
import vern7_dense_ref as V  # noqa: E402
from helpers import glorot_theta, theta_scenario1_init  # noqa: E402


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


RBF3 = ("rbf", "rbf", "rbf")
FORMS = ["lv0", "lv1", "lv2", "seir", "node"]


def _case(O, form, N, seed=0):
    """(UDE form, oracle model, theta, u0[d, N], data[n_save, d, N], loss weights, (save_dt, n_save))."""
    ude = _ude()
    rng = np.random.default_rng(seed)
    if form.startswith("lv"):
        rates = int(form[2])
        acts = ("rbf", "rbf", "tanh") if rates == 2 else RBF3
        chain = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in ((2, 5, acts[0]), (5, 5, acts[1]), (5, 5, acts[2]))], ude.FastDense(5, 2))
        f = ude.LotkaVolterraUDE(chain, trainable_rates=rates)
        m = O.lv_model((2, 5, 5, 5, 2), acts + ("identity",), n_prefix=rates)
        theta = np.concatenate([[1.3, 1.8][2 - rates:] if rates else [], glorot_theta((2, 5, 5, 5, 2), seed=2)]).astype(np.float64)
        if rates == 1:
            theta[0] = 1.7
        u0 = np.stack([rng.uniform(0.2, 1.0, N), rng.uniform(2.0, 5.0, N)])
        y = rng.uniform(0.5, 4.0, (31, 2, N))
        return f, m, theta, u0, y, np.ones(2), (0.1, 31)
    if form == "seir":
        chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
        f = ude.SEIRExposureUDE(chain)
        m = O.seir_model()
        theta = 0.5 * glorot_theta((3, 64, 64, 1), seed=4).astype(np.float64)
        u0 = np.tile(np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])[:, None], (1, N))
        u0[2] *= rng.uniform(0.5, 1.5, N)
        y = O.solve_fixed(m, 0.9 * theta, u0[:, 0], 0.25, 84, save_every=4)[:, :, None] * rng.uniform(0.9, 1.1, (22, 7, N))
        return f, m, theta, u0, y, np.array([0, 1, 1, 1, 0, 0, 0.0]), (1.0, 22)
    chain = ude.FastChain(ude.FastDense(2, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 2))
    f = ude.NeuralODE(chain)
    m = O.make_model(O.MODEL_NODE, 2, (2, 16, 16, 2), ("tanh", "tanh", "identity"))
    theta = glorot_theta((2, 16, 16, 2), seed=6).astype(np.float64)
    u0 = rng.uniform(-1.0, 1.0, (2, N))
    y = rng.uniform(-1.0, 1.0, (31, 2, N))
    return f, m, theta, u0, y, np.ones(2), (0.1, 31)


def _solver(f, grid, N, dtype, w, tol=1e-6, dense=True, sensealg=None, adaptive=True, max_steps=1024):
    ude = _ude()
    sdt, ns = grid
    kw = dict(max_trajectories=N, dtype=dtype, loss_weights=list(w), alg=ude.Vern7(dense=dense), sensealg=sensealg or ude.ForwardDiffSensitivity())
    if adaptive:
        return ude.UDESolver(f, 0.0, sdt, ns - 1, 1, adaptive=True, abstol=tol, reltol=tol, max_steps=max_steps, **kw)
    return ude.UDESolver(f, 0.0, sdt / 2, 2 * (ns - 1), 2, **kw)


def _reference(O, m, theta, u0, y, w, grid, tol=1e-6):
    """fp64 reference: loss, grad_theta, grad_u0[d, N], saved states[n_save, d, N], accepted steps[N]."""
    sdt, ns = grid
    L, G, GU, OUT, NS = 0.0, np.zeros(len(theta)), np.zeros_like(u0), np.zeros((ns,) + u0.shape), []
    for k in range(u0.shape[1]):
        out, rec = V.dense_record(O, m, theta, u0[:, k], 0.0, sdt, ns, tol, tol)
        g, gu = DD.adjoint_dense_steps(O, m, theta, rec, 0.0, sdt, ns, 2 * w * (out - y[:, :, k]))
        L += float((w * (out - y[:, :, k]) ** 2).sum())
        G += g
        GU[:, k] = gu
        OUT[:, :, k] = out
        NS.append(len(rec["hstep"]))
    return L, G, GU, OUT, np.array(NS)


def _run(solver, theta, u0, y, dtype, l2=True):
    npd = np.float64 if dtype == torch.float64 else np.float32
    solver.set_params(torch.from_numpy(np.asarray(theta, npd)).cuda())
    status = torch.full((u0.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(np.asarray(u0, npd)).cuda(), status=status)
    if l2:
        loss, g, gu = solver.adjoint_l2(torch.from_numpy(np.asarray(y, npd)).cuda(), want_grad_u0=True)
        loss = float(loss)
    else:
        g, gu = solver.adjoint(torch.from_numpy(np.asarray(y, npd)).cuda(), want_grad_u0=True)
        loss = None
    torch.cuda.synchronize()
    return out.cpu().numpy(), loss, g.cpu().numpy(), gu.cpu().numpy(), status.cpu().numpy()


@pytest.mark.parametrize("form", FORMS)
def test_f64_vs_reference(O, form):
    N = 5
    f, m, theta, u0, y, w, grid = _case(O, form, N)
    solver = _solver(f, grid, N, torch.float64, w)
    out, loss, g, gu, status = _run(solver, theta, u0, y, torch.float64)
    L, G, GU, OUT, NS = _reference(O, m, theta, u0, y, w, grid)
    assert (status == 0).all()
    assert NS.mean() < grid[1] - 1 or form == "seir"   # fewer steps than save points: the saves come from the interpolant
    scale = np.abs(OUT).max(axis=(0, 2), keepdims=True) + 1.0
    e_out = (np.abs(out - OUT) / scale).max()
    e_g = np.linalg.norm(g - G) / np.linalg.norm(G)
    e_gu = np.abs(gu - GU).max() / np.abs(GU).max()
    print(f"f64 {form}: states {e_out:.2e} loss {abs(loss - L) / abs(L):.2e} grad {e_g:.2e} grad_u0 {e_gu:.2e}")
    # measured on an H100: states <= 1.4e-13 (SEIR, states of 1.4e7 over 21 days: 1.3e-12); loss, grad_theta, grad_u0 <= 3.4e-13
    assert e_out <= 1e-12 * (10 if form == "seir" else 1)
    assert abs(loss - L) <= 1e-9 * abs(L)
    assert e_g <= 1e-9 and e_gu <= 1e-9
    l_out = float((w[None, :, None] * (out - y) ** 2).sum())
    assert abs(loss - l_out) <= 1e-13 * abs(l_out)   # the loss reported is that of the handle's own returned states
    solver.close()


@pytest.mark.parametrize("form", ["lv1", "node", "seir"])
def test_f32_vs_f64_reference(O, form):
    N = 37
    f, m, theta, u0, y, w, grid = _case(O, form, N)
    tol = 1e-5 if form != "seir" else 1e-4
    theta = theta.astype(np.float32).astype(np.float64)
    u0 = u0.astype(np.float32).astype(np.float64)
    y = y.astype(np.float32).astype(np.float64)
    solver = _solver(f, grid, N, torch.float32, w, tol=tol)
    out, loss, g, gu, status = _run(solver, theta, u0, y, torch.float32)
    L, G, GU, OUT, _ = _reference(O, m, theta, u0, y, w, grid, tol=tol)
    assert (status == 0).all()
    scale = np.abs(OUT).max(axis=(0, 2), keepdims=True) + 1.0
    e_out = (np.abs(out - OUT) / scale).max()
    e_g = np.linalg.norm(g - G) / np.linalg.norm(G)
    e_gu = np.abs(gu - GU).max() / np.abs(GU).max()
    print(f"f32 {form}: states {e_out:.2e} loss {abs(loss - L) / abs(L):.2e} grad {e_g:.2e} grad_u0 {e_gu:.2e}")
    # the bounds the fp32 dense-output handle is held to on its adaptive grid.  Measured on an H100: states <= 1.5e-5 of scale, loss
    # <= 2.3e-7, grad_theta <= 1.1e-6, grad_u0 <= 3.5e-6
    assert e_out <= 1e-4
    assert abs(loss - L) <= 1e-5 * abs(L)
    assert e_g <= 2e-5 and e_gu <= 2e-5
    solver.close()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_forward_is_the_dense_output_forward_and_fused_equals_unfused(O, dtype):
    """Saved states and status are bitwise those of the Vern7(dense=True) + InterpolatingAdjoint handle (the same forward kernel
    and record), the gradient is not that handle's, and the fused L2 equals the plain adjoint fed 2 w (out - data)."""
    ude = _ude()
    N = 9
    for form in ("lv1", "seir"):
        f, m, theta, u0, y, w, grid = _case(O, form, N, seed=3)
        tol = 1e-6 if dtype == torch.float64 else (1e-5 if form != "seir" else 1e-4)
        dd = _solver(f, grid, N, dtype, w, tol=tol)
        ia = _solver(f, grid, N, dtype, w, tol=tol, sensealg=ude.InterpolatingAdjoint())
        r_dd = _run(dd, theta, u0, y, dtype)
        r_ia = _run(ia, theta, u0, y, dtype)
        assert np.array_equal(r_dd[0], r_ia[0]) and np.array_equal(r_dd[4], r_ia[4])
        assert abs(r_dd[1] - r_ia[1]) <= (1e-13 if dtype == torch.float64 else 1e-6) * abs(r_ia[1])
        assert not np.array_equal(r_dd[2], r_ia[2])
        npd = r_dd[0].dtype
        cot = (2 * w.astype(npd))[None, :, None] * (r_dd[0] - y.astype(npd))
        r_un = _run(dd, theta, u0, cot, dtype, l2=False)
        assert np.array_equal(r_un[0], r_dd[0])
        eps = 1e-13 if dtype == torch.float64 else 1e-6
        assert np.linalg.norm(r_un[2] - r_dd[2]) <= eps * np.linalg.norm(r_dd[2])
        assert np.abs(r_un[3] - r_dd[3]).max() <= eps * np.abs(r_dd[3]).max()
        dd.close()
        ia.close()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_each_trajectory_alone_and_run_to_run(O, dtype):
    """N not a multiple of 32 with different step counts within a warp (so lanes without a save inside their step run the extra
    stages with zero weight beside lanes that have one): states, status and grad_u0 of a trajectory are bitwise those of the
    trajectory solved alone, and two runs are bitwise identical."""
    N = 40
    f, m, theta, u0, y, w, grid = _case(O, "lv1", N, seed=5)
    u0[:, ::3] *= 1.7
    solver = _solver(f, grid, N, dtype, w, tol=1e-6 if dtype == torch.float64 else 1e-5)
    a = _run(solver, theta, u0, y, dtype)
    b = _run(solver, theta, u0, y, dtype)
    for x, z in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(z))
    assert (a[4] == 0).all()
    if dtype == torch.float64:
        ns = np.array([len(V.dense_record(O, m, theta, u0[:, k], 0.0, grid[0], grid[1], 1e-6, 1e-6)[1]["hstep"]) for k in range(N)])
        assert len(set(ns[:32])) > 1   # mixed step counts within the first warp
    for k in (0, 3, 17, 39):
        s = _run(solver, theta, u0[:, k:k + 1], y[:, :, k:k + 1], dtype)
        assert np.array_equal(s[0][:, :, 0], a[0][:, :, k])
        assert s[4][0] == a[4][k]
        assert np.array_equal(s[3][:, 0], a[3][:, k])
    solver.close()


def test_f64_max_steps_status_and_nan(O):
    """A trajectory that needs more than max_steps accepted steps reports status 2, NaN at the save points it did not reach and so a
    NaN loss (as the tstops kernels do); the states, status and grad_u0 of the others are bitwise those of a handle with room."""
    N = 12
    f, m, theta, u0, y, w, grid = _case(O, "lv1", N, seed=7)
    u0[:, ::2] *= 1.7
    ns = np.array([len(V.dense_record(O, m, theta, u0[:, k], 0.0, grid[0], grid[1], 1e-6, 1e-6)[1]["hstep"]) for k in range(N)])
    cap = int(np.sort(ns)[N // 2 - 1])
    short = ns > cap
    assert short.any() and not short.all(), ns
    roomy = _solver(f, grid, N, torch.float64, w)
    tight = _solver(f, grid, N, torch.float64, w, max_steps=cap)
    r = _run(roomy, theta, u0, y, torch.float64)
    t = _run(tight, theta, u0, y, torch.float64)
    assert np.array_equal(t[4], np.where(short, 2, 0)), (t[4], ns, cap)
    assert np.isnan(t[1])
    assert np.isnan(t[0][-1][:, short]).all() and np.isfinite(t[0][0]).all()
    assert np.array_equal(t[0][:, :, ~short], r[0][:, :, ~short])
    assert np.array_equal(t[3][:, ~short], r[3][:, ~short])
    assert np.isnan(t[3][:, short]).all()
    roomy.close()
    tight.close()


class _WithFlag:
    """The C library with `flag` or-ed into every descriptor it is asked to create a handle for."""

    def __init__(self, L, flag):
        self._L, self._flag = L, flag

    def b200ude_create(self, d, h):
        d._obj.flags |= self._flag
        return self._L.b200ude_create(d, h)

    def __getattr__(self, name):
        return getattr(self._L, name)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_fixed_grid_with_the_flag_is_the_plain_discrete_kernel(O, dtype, monkeypatch):
    """adaptive = 0: the saves are step ends, the flag is accepted and everything is bitwise the handle without it (which is what
    Vern7(dense=True) with ForwardDiffSensitivity creates on a fixed grid)."""
    from universal_differential_equations_b200 import _lib, sciml
    N = 7
    f, m, theta, u0, y, w, grid = _case(O, "lv1", N, seed=2)
    plain = _solver(f, grid, N, dtype, w, adaptive=False)
    L = _lib.lib()
    monkeypatch.setattr(sciml._lib, "lib", lambda: _WithFlag(L, _lib.FLAG_DISCRETE_DENSE))
    flagged = _solver(f, grid, N, dtype, w, adaptive=False)
    monkeypatch.undo()
    assert isinstance(flagged._L, _WithFlag)
    a = _run(plain, theta, u0, y, dtype)
    b = _run(flagged, theta, u0, y, dtype)
    for x, z in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(z))
    plain.close()
    flagged.close()


def test_refused_combinations_name_the_flag():
    ude = _ude()
    from universal_differential_equations_b200 import _lib
    chain = ude.FastChain(ude.FastDense(1, 10, ude.tanh), ude.FastDense(10, 1))
    with pytest.raises(_lib.B200UDEError, match="B200UDE_FLAG_DISCRETE_DENSE") as e:
        ude.UDESolver(ude.FisherKPPUDE(chain, 26), 0.0, 0.5, 10, 1, alg=ude.Vern7(dense=True), sensealg=ude.ForwardDiffSensitivity(), adaptive=True)
    assert e.value.code == _lib.EUNSUPPORTED


def test_scenario_1_verbatim_f64_on_the_scripts_own_step_sequence(golden):
    """scenario_1.jl:84-87,91-94,114 as written, in Float64: solve(prob, Vern7(); saveat = 0.1, abstol = reltol = 1e-6,
    sensealg = ForwardDiffSensitivity()) stepping freely with interpolated saves, inside sciml_train(loss, theta_init, ADAM(0.1)),
    against the stored losses[0..5]: the bounds of the CPU reference (tests/test_vern7_dense_discrete_oracle.py: 1e-6 up to
    losses[4], 5e-6 at losses[5], where it measures 3.1e-6)."""
    ude = _ude()
    g = golden["scenario_1"]
    chain = ude.FastChain(*[ude.FastDense(a, b, "rbf") for a, b in ((2, 5), (5, 5), (5, 5))], ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain)
    X = torch.from_numpy(g["X"].astype(np.float64)).cuda()
    prob = ude.ODEProblem(f, g["X"][:, 0].astype(np.float64), (0.0, 3.0), None)
    seen = []

    def loss(th):
        pred = ude.concrete_solve(prob, ude.Vern7(dense=True), p=th, saveat=0.1, abstol=1e-6, reltol=1e-6,
                                  sensealg=ude.ForwardDiffSensitivity(), dtype=torch.float64)
        return ((X - pred) ** 2).sum()

    def cb(th, l):
        seen.append(l)
        return len(seen) >= 6
    ude.sciml_train(loss, torch.from_numpy(theta_scenario1_init(g)).cuda(), ude.ADAM(0.1), cb=cb, maxiters=10)
    ref = g["losses"][:6]
    err = np.abs(np.array(seen) - ref) / ref
    print("scenario 1 losses[0..5] relative:", ["%.1e" % e for e in err])
    assert err[0] <= 1e-10 and np.all(err[:5] <= 1e-6) and err[5] <= 5e-6, (seen, ref)
