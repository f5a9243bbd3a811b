"""Discrete adjoint (sensealg = ForwardDiffSensitivity) of fixed-step Tsit5 / Vern7 and adaptive Vern7 on the runtime-shape
kernels (discrete_adjoint.cuh), fp32 and fp64: against the fp64 reference discrete adjoint (tests/discrete_ref.py, pinned to
torch autograd in tests/test_discrete_adjoint_oracle.py), the LV scripts' calls as written against the reference's stored loss
histories, record consistency, determinism, trajectory isolation and the fp32 entry points."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import discrete_ref as R  # noqa: E402
from helpers import glorot_theta, theta_scenario1_init  # noqa: E402


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


RBF3 = ("rbf", "rbf", "rbf")


def _case(O, form, N, seed=0):
    """(UDE form, oracle model, theta, u0[d, N], data factory, loss weights, (save_dt, n_save))."""
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


def _solver(f, stepping, grid, N, dtype, w, tol=1e-6):
    ude = _ude()
    sdt, ns = grid
    kw = dict(max_trajectories=N, sensealg=ude.ForwardDiffSensitivity(), dtype=dtype, loss_weights=list(w))
    if stepping == "adaptive":
        return ude.UDESolver(f, 0.0, sdt, ns - 1, 1, alg=ude.Vern7(), adaptive=True, abstol=tol, reltol=tol, max_steps=1024, **kw)
    alg = ude.Vern7() if stepping == "vern7" else ude.Tsit5()
    return ude.UDESolver(f, 0.0, sdt / 2, 2 * (ns - 1), 2, alg=alg, **kw)


def _reference(O, m, theta, u0, y, w, stepping, grid, tol=1e-6):
    """fp64 reference: loss, grad_theta, grad_u0[d, N], saved states[n_save, d, N]."""
    sdt, ns = grid
    L, G, GU, OUT = 0.0, np.zeros(len(theta)), np.zeros_like(u0), np.zeros((ns,) + u0.shape)
    for k in range(u0.shape[1]):
        if stepping == "adaptive":
            out, rec = R.vern7_adaptive_record(O, m, theta, u0[:, k], 0.0, sdt, ns, tol, tol)
            ustep, solver = rec["ustep"], R.VERN7
        else:
            solver = R.VERN7 if stepping == "vern7" else R.TSIT5
            rec = R.fixed_record(2 * (ns - 1), sdt / 2, 2)
            out, ustep = R.solve_steps(O, m, theta, u0[:, k], rec, solver)
        g, gu = R.adjoint_steps(O, m, theta, ustep, rec, solver, 2 * w * (out - y[:, :, k]))
        L += float((w * (out - y[:, :, k]) ** 2).sum())
        G += g
        GU[:, k] = gu
        OUT[:, :, k] = out
    return L, G, GU, OUT


def _run(solver, theta, u0, y, dtype):
    npd = np.float64 if dtype == torch.float64 else np.float32
    solver.set_params(torch.from_numpy(np.asarray(theta, npd)).cuda())
    status = torch.full((u0.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(np.asarray(u0, npd)).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(np.asarray(y, npd)).cuda(), want_grad_u0=True)
    torch.cuda.synchronize()
    return out.cpu().numpy(), float(loss), g.cpu().numpy(), gu.cpu().numpy(), status.cpu().numpy()


FORMS = ["lv0", "lv1", "lv2", "seir", "node"]


@pytest.mark.parametrize("stepping", ["vern7", "tsit5", "adaptive"])
@pytest.mark.parametrize("form", FORMS)
def test_f64_discrete_adjoint_vs_reference(O, form, stepping):
    N = 5
    f, m, theta, u0, y, w, grid = _case(O, form, N)
    solver = _solver(f, stepping, grid, N, torch.float64, w)
    out, loss, g, gu, status = _run(solver, theta, u0, y, torch.float64)
    L, G, GU, OUT = _reference(O, m, theta, u0, y, w, stepping, grid)
    assert (status == 0).all()
    bound = 1e-6 if stepping == "adaptive" else 1e-10   # adaptive: the kernel's own step sequence, same controller
    scale = np.abs(OUT).max(axis=(0, 2), keepdims=True) + 1.0
    assert np.all(np.abs(out - OUT) <= bound * scale)
    assert abs(loss - L) <= bound * abs(L)
    assert np.linalg.norm(g - G) <= bound * np.linalg.norm(G)
    assert np.abs(gu - GU).max() <= bound * np.abs(GU).max()
    # the loss the adjoint reports is the one of the handle's own saved states (Vern7: no Tsit5 re-solve involved)
    l_out = float((w[None, :, None] * (out - y) ** 2).sum())
    assert abs(loss - l_out) <= 1e-13 * abs(l_out)
    if stepping == "vern7" and form in ("lv1", "node"):
        # directional finite difference of the GPU loss itself
        v = np.random.default_rng(3).standard_normal(len(theta))
        v /= np.linalg.norm(v)
        eps = 1e-5
        lp = _run(solver, theta + eps * v, u0, y, torch.float64)[1]
        lm = _run(solver, theta - eps * v, u0, y, torch.float64)[1]
        fd = (lp - lm) / (2 * eps)
        assert abs(fd - g @ v) <= 1e-7 * max(abs(fd), 1e-3 * np.linalg.norm(g)), (fd, g @ v)
    solver.close()


@pytest.mark.parametrize("stepping", ["vern7", "adaptive"])
@pytest.mark.parametrize("form", FORMS)
def test_f32_discrete_adjoint_vs_f64_reference(O, form, stepping):
    N = 8 if form == "seir" else 40
    f, m, theta, u0, y, w, grid = _case(O, form, N, seed=1)
    tol = 1e-5 if form == "seir" else 1e-6   # SEIR in fp32: populations of 1.4e7 leave an fp32 state ~8 ulp of room at 1e-6
    theta, u0, y = (a.astype(np.float32) for a in (theta, u0, y))
    solver = _solver(f, stepping, grid, N, torch.float32, w, tol)
    out, loss, g, gu, status = _run(solver, theta, u0, y, torch.float32)
    L, G, GU, _ = _reference(O, m, theta.astype(np.float64), u0.astype(np.float64), y.astype(np.float64), w, stepping, grid, tol)
    assert (status == 0).all()
    assert abs(loss - L) <= 1e-4 * abs(L)
    assert np.linalg.norm(g - G) <= 2e-3 * np.linalg.norm(G)
    assert np.abs(gu - GU).max() <= 2e-3 * np.abs(GU).max()
    # the loss the adjoint reports is the one of the handle's own saved states
    l_out = float((w[None, :, None] * (out.astype(np.float64) - y) ** 2).sum())
    assert abs(loss - l_out) <= 1e-6 * abs(l_out)
    solver.close()


def test_scenario_1_verbatim_f64_reproduces_reference_loss_history(golden):
    """scenario_1.jl:84-87,91-94,114 as written, in Float64: solve(prob, Vern7(); saveat = 0.1, abstol = reltol = 1e-6,
    sensealg = ForwardDiffSensitivity()) inside sciml_train(loss, theta_init, ADAM(0.1)) replays the stored losses[0..5]."""
    ude = _ude()
    g = golden["scenario_1"]
    chain = ude.FastChain(*[ude.FastDense(a, b, "rbf") for a, b in ((2, 5), (5, 5), (5, 5))], ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain)
    X = torch.from_numpy(g["X"].astype(np.float64)).cuda()
    prob = ude.ODEProblem(f, g["X"][:, 0].astype(np.float64), (0.0, 3.0), None)
    seen = []

    def loss(th):
        pred = ude.concrete_solve(prob, ude.Vern7(), p=th, saveat=0.1, abstol=1e-6, reltol=1e-6, sensealg=ude.ForwardDiffSensitivity(),
                                  dtype=torch.float64)
        return ((X - pred) ** 2).sum()

    def cb(th, l):
        seen.append(l)
        return len(seen) >= 6
    ude.sciml_train(loss, torch.from_numpy(theta_scenario1_init(g)).cuda(), ude.ADAM(0.1), cb=cb, maxiters=10)
    ref = g["losses"][:6]
    assert np.all(np.abs(np.array(seen) - ref) <= 2e-6 * ref), (seen, ref)


def test_scenario_2_kat9_f64_multiple_shooting_through_vern7_forwarddiff(golden):
    """KAT-9 through the script's own call (scenario_2.jl:57-72,106-123): theta = [delta; U], five shooting segments of 1.2 solved
    as one 5-trajectory ensemble with Vern7 @ 1e-6 and ForwardDiffSensitivity in Float64, loss = sum over segments of
    sum (x data - x_hat)^2 + |y(end) - y_hat(end)|, plus 1e-3 mean(theta[2:end]^2); ADAM(0.1) replays the stored losses[0..5]."""
    ude = _ude()
    g = golden["scenario_2"]
    t, Xd = g["t"], g["X"]
    ty = np.arange(t[0], t[-1] + 1e-9, 6 / 5)
    segs = [np.where((t >= ty[i] - 1e-9) & (t <= ty[i + 1] + 1e-9))[0] for i in range(len(ty) - 1)]
    chain = ude.FastChain(*[ude.FastDense(a, b, "rbf") for a, b in ((2, 5), (5, 5), (5, 5))], ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain, trainable_rates=1)
    u0s = np.stack([Xd[:, s[0]] for s in segs], axis=1).astype(np.float64)
    xs = torch.from_numpy(np.stack([Xd[0, s] for s in segs], axis=1).astype(np.float64)).cuda()   # [13, 5]
    y1 = torch.from_numpy(np.array([Xd[1, s[-1]] for s in segs], np.float64)).cuda()
    prob = ude.EnsembleProblem(ude.ODEProblem(f, u0s[:, 0], (0.0, 1.2), None), u0s)
    seen = []

    def loss(th):
        pred = ude.concrete_solve(prob, ude.Vern7(), p=th, saveat=0.1, abstol=1e-6, reltol=1e-6, sensealg=ude.ForwardDiffSensitivity(),
                                  dtype=torch.float64)   # [13, 2, 5]
        return ((xs - pred[:, 0, :]) ** 2).sum() + (y1 - pred[-1, 1, :]).abs().sum() + 1e-3 * (th[1:] ** 2).mean()

    def cb(th, l):
        seen.append(l)
        return len(seen) >= 6
    ude.sciml_train(loss, torch.from_numpy(g["theta_init"].astype(np.float64)).cuda(), ude.ADAM(0.1), cb=cb, maxiters=10)
    ref = g["losses"][:6]
    assert np.all(np.abs(np.array(seen) - ref) <= 2e-6 * ref), (seen, ref)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_adaptive_determinism_and_trajectory_isolation(O, dtype):
    """Repeated calls are bitwise identical; each trajectory's saved states, status and grad_u0 equal the same trajectory solved
    alone, whatever its warp neighbours (here: neighbours with other step counts)."""
    N = 70
    f, m, theta, u0, y, w, grid = _case(O, "lv1", N, seed=2)
    u0[:, 1::3] *= 1.6   # different dynamics -> different accepted-step counts within each warp
    solver = _solver(f, "adaptive", grid, N, dtype, w)
    a = _run(solver, theta, u0, y, dtype)
    b = _run(solver, theta, u0, y, dtype)
    for x, z in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(z))
    for k in (0, 1, 33, 69):
        one = _solver(f, "adaptive", grid, 1, dtype, w)
        o1, _, _, gu1, st1 = _run(one, theta, u0[:, k:k + 1].copy(), y[:, :, k:k + 1].copy(), dtype)
        assert np.array_equal(o1[:, :, 0], a[0][:, :, k]) and st1[0] == a[4][k]
        assert np.array_equal(gu1[:, 0], a[3][:, k]), k
        one.close()
    solver.close()


def test_f32_fixed_vern7_entry_points_bitwise(monkeypatch):
    """fp32 fixed-step Vern7 with the discrete adjoint: train_adam through the CUDA graph equals the same iterations launched one
    by one, and loss_gradient_host equals the device-pointer path, bit for bit."""
    ude = _ude()
    import oracle.oracle as O
    N = 300
    f, m, theta, u0, y, w, grid = _case(O, "lv1", N, seed=4)
    th32, u32, y32 = theta.astype(np.float32), u0.astype(np.float32), y.astype(np.float32)
    hist = {}
    for graph in ("1", "0"):
        monkeypatch.setenv("B200UDE_TRAIN_GRAPH", graph)
        s = _solver(f, "vern7", grid, N, torch.float32, w)
        s.set_params(torch.from_numpy(th32).cuda())
        s.adam_reset()
        l = s.train_adam(ude.ADAM(0.01), torch.from_numpy(u32).cuda(), torch.from_numpy(y32).cuda(), 8).cpu().numpy()
        hist[graph] = (l, s.get_params().cpu().numpy())
        s.close()
    assert np.array_equal(hist["1"][0], hist["0"][0]) and np.array_equal(hist["1"][1], hist["0"][1])
    assert np.all(np.isfinite(hist["1"][0]))
    s = _solver(f, "vern7", grid, N, torch.float32, w)
    _, loss_d, g_d, gu_d, _ = _run(s, th32, u32, y32, torch.float32)
    gu_h = np.empty_like(u32)
    loss_h, g_h, _ = s.loss_gradient_host(th32, u32, y32, grad_u0=gu_h)
    assert np.float32(loss_h) == np.float32(loss_d)
    assert np.array_equal(g_h, g_d) and np.array_equal(gu_h, gu_d)
    s.close()
