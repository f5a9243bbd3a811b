"""Vern7 with its lazy dense output (B200UDE_FLAG_VERN7_DENSE, `Vern7(dense=True)`) on the GPU, fp64 and fp32: forward and
interpolating adjoint against the fp64 reference (tests/vern7_dense_ref.py, pinned on the CPU to the reference's artefacts and an
error-controlled backward solve), the scenario 1 and SEIR script calls as written, trajectory isolation, determinism, and that
the flag selects the new path and moves nothing else."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import vern7_dense_ref as V  # noqa: E402
from helpers import glorot_theta  # noqa: E402


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


RBF3 = ("rbf", "rbf", "rbf")


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


def _solver(f, stepping, grid, N, dtype, w, tol=1e-6, dense=True, alg=None):
    ude = _ude()
    sdt, ns = grid
    alg = alg or ude.Vern7(dense=dense)
    kw = dict(max_trajectories=N, dtype=dtype, loss_weights=list(w), alg=alg)
    if stepping == "adaptive":
        return ude.UDESolver(f, 0.0, sdt, ns - 1, 1, adaptive=True, abstol=tol, reltol=tol, max_steps=1024, **kw)
    return ude.UDESolver(f, 0.0, sdt / 2, 2 * (ns - 1), 2, **kw)


def _reference(O, m, theta, u0, y, w, stepping, grid, tol=1e-6):
    """fp64 reference: loss, grad_theta, grad_u0[d, N], saved states[n_save, d, N]."""
    sdt, ns = grid
    L, G, GU, OUT = 0.0, np.zeros(len(theta)), np.zeros_like(u0), np.zeros((ns,) + u0.shape)
    for k in range(u0.shape[1]):
        if stepping == "adaptive":
            out, rec = V.dense_record(O, m, theta, u0[:, k], 0.0, sdt, ns, tol, tol)
        else:
            out, rec = V.fixed_record(O, m, theta, u0[:, k], 0.0, sdt / 2, 2 * (ns - 1), 2)
        g, gu = V.replay_adjoint(O, m, theta, rec, 0.0, sdt, ns, 2 * w * (out - y[:, :, k]))
        L += float((w * (out - y[:, :, k]) ** 2).sum())
        G += g
        GU[:, k] = gu
        OUT[:, :, k] = out
    return L, G, GU, OUT


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


FORMS = ["lv0", "lv1", "lv2", "seir", "node"]


@pytest.mark.parametrize("stepping", ["fixed", "adaptive"])
@pytest.mark.parametrize("form", FORMS)
def test_f64_vern7_dense_vs_reference(O, form, stepping):
    N = 5
    f, m, theta, u0, y, w, grid = _case(O, form, N)
    solver = _solver(f, stepping, grid, N, torch.float64, w)
    out, loss, g, gu, status = _run(solver, theta, u0, y, torch.float64)
    L, G, GU, OUT = _reference(O, m, theta, u0, y, w, stepping, grid)
    assert (status == 0).all()
    scale = np.abs(OUT).max(axis=(0, 2), keepdims=True) + 1.0
    e_out = (np.abs(out - OUT) / scale).max()
    e_g = np.linalg.norm(g - G) / np.linalg.norm(G)
    e_gu = np.abs(gu - GU).max() / np.abs(GU).max()
    print(f"f64 {form} {stepping}: states {e_out:.2e} loss {abs(loss - L) / abs(L):.2e} grad {e_g:.2e} grad_u0 {e_gu:.2e}")
    # measured on an H100: states <= 2.8e-16 fixed, <= 1.3e-12 adaptive (SEIR); loss, grad_theta, grad_u0 <= 8.2e-14
    assert e_out <= (1e-11 if stepping == "adaptive" else 1e-14)
    assert abs(loss - L) <= 1e-12 * abs(L)
    assert e_g <= 1e-12 and e_gu <= 1e-12
    # the loss the adjoint reports is the one of the handle's own returned states
    l_out = float((w[None, :, None] * (out - y) ** 2).sum())
    assert abs(loss - l_out) <= 1e-13 * abs(l_out)
    solver.close()


@pytest.mark.parametrize("stepping", ["fixed", "adaptive"])
@pytest.mark.parametrize("form", ["lv1", "node", "seir"])
def test_f32_vern7_dense_vs_f64_reference(O, form, stepping):
    N = 37
    f, m, theta, u0, y, w, grid = _case(O, form, N)
    tol = 1e-5 if form != "seir" else 1e-4
    theta = theta.astype(np.float32).astype(np.float64)
    u0 = u0.astype(np.float32).astype(np.float64)
    y = y.astype(np.float32).astype(np.float64)
    solver = _solver(f, stepping, grid, N, torch.float32, w, tol=tol)
    out, loss, g, gu, status = _run(solver, theta, u0, y, torch.float32)
    L, G, GU, OUT = _reference(O, m, theta, u0, y, w, stepping, grid, tol=tol)
    assert (status == 0).all()
    scale = np.abs(OUT).max(axis=(0, 2), keepdims=True) + 1.0
    e_out = (np.abs(out - OUT) / scale).max()
    e_g = np.linalg.norm(g - G) / np.linalg.norm(G)
    e_gu = np.abs(gu - GU).max() / np.abs(GU).max()
    print(f"f32 {form} {stepping}: states {e_out:.2e} loss {abs(loss - L) / abs(L):.2e} grad {e_g:.2e} grad_u0 {e_gu:.2e}")
    # measured on an H100: states <= 4.5e-7 of scale fixed, <= 1.5e-5 adaptive; loss and grad_theta <= 8.4e-7, grad_u0 <= 2e-6
    adaptive = stepping == "adaptive"
    assert e_out <= (1e-4 if adaptive else 5e-6)
    assert abs(loss - L) <= 1e-5 * abs(L)
    assert e_g <= 2e-5 and e_gu <= 2e-5
    l_out = float((w[None, :, None] * (out.astype(np.float64) - y) ** 2).sum())
    assert abs(loss - l_out) <= 1e-4 * abs(l_out)
    solver.close()


def test_f64_scenario1_call_as_written(O, golden):
    """solve(prob, Vern7(); saveat = 0:0.05:3, abstol = reltol = 1e-6) in Float64 (scenario_1.jl:41,84-85) with saves from the
    interpolant, against the reference's stored X-hat (bounds of the CPU reference: round-off up to t = 2.85, 5e-7 overall) and the
    fp64 reference; the gradient against the reference's replay."""
    ude = _ude()
    g = golden["scenario_1"]
    chain = ude.FastChain(*[ude.FastDense(a, b, ude.rbf) for a, b in ((2, 5), (5, 5), (5, 5))], ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain)
    m = O.lv_model((2, 5, 5, 5, 2), RBF3 + ("identity",))
    theta = g["theta_trained"].astype(np.float64)
    N = 3
    u0 = np.repeat(g["X"][:, :1], N, axis=1).astype(np.float64)
    y = np.random.default_rng(0).normal(size=(61, 2, N))
    solver = ude.UDESolver(f, 0.0, 0.05, 60, 1, max_trajectories=N, alg=ude.Vern7(dense=True), adaptive=True, abstol=1e-6, reltol=1e-6,
                           max_steps=512, dtype=torch.float64)
    out, loss, gth, gu, status = _run(solver, theta, u0, y, torch.float64)
    assert (status == 0).all()
    err = np.abs(out[:, :, 0].T - g["Xhat"]).max(axis=0)
    print(f"scenario 1: X-hat up to t=2.85 {err[:58].max():.2e}, overall {err.max():.2e}")
    assert err[:58].max() <= 1e-11 and err.max() <= 5e-7
    L, G, GU, OUT = _reference(O, m, theta, u0, y, np.ones(2), "adaptive", (0.05, 61))
    e_ref = np.abs(out - OUT).max()
    print(f"scenario 1: against the fp64 reference {e_ref:.2e}")
    assert e_ref <= 1e-11   # measured 3.1e-12
    assert np.linalg.norm(gth - G) <= 1e-11 * np.linalg.norm(G)
    solver.close()


def test_f64_seir_script_call_as_written(O):
    """seir_exposure.jl:137-141 with the flag: concrete_solve(prob_nn, Vern7(dense=True), u0, theta; saveat = 0:21, abstol = reltol
    = 1e-6, sensealg = InterpolatingAdjoint(...)) in Float64 through the torch-facing call surface, the loss on E, I, R (:146);
    forward and gradient against the fp64 reference replay, and adjoint_l2's loss equal to the loss of the returned states."""
    ude = _ude()
    ann = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    p = ude.initial_params(ann, np.random.default_rng(0)).astype(np.float64)
    u0 = np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])
    w = np.array([0, 1, 1, 1, 0, 0, 0.0])
    m = O.seir_model()
    data = O.solve_fixed(m, 0.9 * p, u0, 0.25, 84, save_every=4)
    prob = ude.ODEProblem(ude.SEIRExposureUDE(ann), u0, (0.0, 21.0), None)
    th = torch.tensor(p, device="cuda", requires_grad=True)
    pred = ude.concrete_solve(prob, ude.Vern7(dense=True), p=th, saveat=np.arange(0.0, 22.0), abstol=1e-6, reltol=1e-6,
                              sensealg=ude.InterpolatingAdjoint(), dtype=torch.float64)
    wt = torch.tensor(w, device="cuda")
    loss = (wt[:, None] * (pred - torch.tensor(data.T, device="cuda")) ** 2).sum()
    loss.backward()
    out_ref, rec = V.dense_record(O, m, p, u0, 0.0, 1.0, 22, 1e-6, 1e-6)
    g_ref, _ = V.replay_adjoint(O, m, p, rec, 0.0, 1.0, 22, 2 * w * (out_ref - data))
    scale = np.abs(out_ref).max(axis=0) + 1.0
    e_out = (np.abs(pred.detach().cpu().numpy().T - out_ref) / scale).max()
    e_g = np.linalg.norm(th.grad.cpu().numpy() - g_ref) / np.linalg.norm(g_ref)
    print(f"SEIR script call: states {e_out:.2e} grad {e_g:.2e}")
    assert e_out <= 1e-10 and e_g <= 1e-10   # measured 1.5e-12 and 2.2e-12
    # the fused entry point on the same handle configuration: its loss is the loss of the states it returned
    solver = ude.UDESolver(ude.SEIRExposureUDE(ann), 0.0, 1.0, 21, 1, max_trajectories=1, alg=ude.Vern7(dense=True), adaptive=True,
                           abstol=1e-6, reltol=1e-6, max_steps=512, loss_weights=list(w), dtype=torch.float64)
    out, l2, g2, _, status = _run(solver, p, u0[:, None], data[:, :, None], torch.float64)
    assert status[0] == 0
    assert abs(l2 - float((w[None, :] * (out[:, :, 0] - data) ** 2).sum())) <= 1e-13 * l2
    assert np.linalg.norm(g2 - g_ref) <= 1e-10 * np.linalg.norm(g_ref)
    solver.close()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_each_trajectory_alone_and_run_to_run(O, dtype):
    """Adaptive: every trajectory's states, status and grad_u0 are bitwise those of the trajectory solved alone (its warp's other
    lanes take other step counts), and two runs are bitwise identical."""
    N = 40
    f, m, theta, u0, y, w, grid = _case(O, "lv1", N, seed=5)
    u0[:, ::3] *= 1.7   # different step counts within a warp
    solver = _solver(f, "adaptive", grid, N, dtype, w, tol=1e-6 if dtype == torch.float64 else 1e-5)
    a = _run(solver, theta, u0, y, dtype)
    b = _run(solver, theta, u0, y, dtype)
    for x, z in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(z))
    assert (a[4] == 0).all()
    for k in (0, 3, 17, 39):
        s = _run(solver, theta, u0[:, k:k + 1], y[:, :, k:k + 1], dtype)
        assert np.array_equal(s[0][:, :, 0], a[0][:, :, k])
        assert s[4][0] == a[4][k]
        assert np.array_equal(s[3][:, 0], a[3][:, k])
    solver.close()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_flag_selects_the_new_path_and_nothing_else(O, dtype):
    """Without the flag a Vern7 handle's interpolating adjoint is, bit for bit, that of a Tsit5 handle with the same u0 and tolerances
    (the re-solve it runs: b200ude.cu launches the same adaptive Tsit5 forward and replay kernels for both on these runtime-shape
    forms), and its forward is the tstops solve; with the flag the adjoint is the dense-output one, and the fused loss is the
    loss of the handle's own states."""
    ude = _ude()
    N = 7
    for form in ("lv1", "node"):
        f, m, theta, u0, y, w, grid = _case(O, form, N, seed=2)
        tol = 1e-6 if dtype == torch.float64 else 1e-5
        v7 = _solver(f, "adaptive", grid, N, dtype, w, tol=tol, dense=False)
        ts5 = _solver(f, "adaptive", grid, N, dtype, w, tol=tol, alg=ude.Tsit5())
        dn = _solver(f, "adaptive", grid, N, dtype, w, tol=tol, dense=True)
        cot = np.random.default_rng(1).standard_normal(y.shape)
        r_v7 = _run(v7, theta, u0, cot, dtype, l2=False)
        r_ts = _run(ts5, theta, u0, cot, dtype, l2=False)
        r_dn = _run(dn, theta, u0, cot, dtype, l2=False)
        assert np.array_equal(r_v7[2], r_ts[2]) and np.array_equal(r_v7[3], r_ts[3])
        assert not np.array_equal(r_dn[2], r_v7[2])
        # the tstops forward of the flag-off handle is the CPU reference's tstops solve; the flag-on one saves by the interpolant
        o_tstops, _, _ = O.solve_adaptive(m, theta.astype(np.float64), u0[:, 0].astype(np.float64), grid[0] * np.arange(grid[1]), tol, tol,
                                          solver=O.VERN7)
        assert np.abs(r_v7[0][:, :, 0] - o_tstops).max() <= (1e-9 if dtype == torch.float64 else 1e-3) * (np.abs(o_tstops).max() + 1)
        l2 = _run(dn, theta, u0, y, dtype)
        l_out = float((w[None, :, None] * (l2[0].astype(np.float64) - y.astype(l2[0].dtype).astype(np.float64)) ** 2).sum())
        assert abs(l2[1] - l_out) <= (1e-13 if dtype == torch.float64 else 1e-5) * abs(l_out)
        for s in (v7, ts5, dn):
            s.close()
