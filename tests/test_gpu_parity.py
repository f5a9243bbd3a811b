"""GPU parity tests: the sm_90a kernels, called through the C ABI, against the CPU oracle.

Tolerances (fp32 kernels; the oracle is evaluated in fp64 and, where stated, fp32):
  trajectories  |out - oracle64| <= 3e-4 * (1 + |oracle|)     (fp32 vs fp64 over 30 Tsit5 steps: ~1.4e-4 rel, SURVEY App. C)
  loss          rel <= 1e-4
  grad_theta    ||g - g_oracle64|| / ||g_oracle64|| <= 2e-3 ; vs the fp32 oracle <= 2e-3 as well (both carry fp32 round-off)
  grad_u0       max-abs rel <= 2e-3
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import theta_scenario1_init, glorot_theta, synthetic_ensemble  # noqa: E402


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _lv32(ude):
    chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
    return ude.LotkaVolterraUDE(chain)


def _lv5(ude, acts=("rbf", "rbf", "rbf"), rates=0):
    chain = ude.FastChain(ude.FastDense(2, 5, acts[0]), ude.FastDense(5, 5, acts[1]), ude.FastDense(5, 5, acts[2]), ude.FastDense(5, 2))
    return ude.LotkaVolterraUDE(chain, trainable_rates=rates)


def _run(solver, theta, u0, data, want_gu0=True):
    th = torch.from_numpy(theta.astype(np.float32)).cuda()
    solver.set_params(th)
    status = torch.full((u0.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(u0).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(data).cuda(), want_grad_u0=want_gu0)
    torch.cuda.synchronize()
    return out.cpu().numpy(), float(loss), g.cpu().numpy(), (gu.cpu().numpy() if gu is not None else None), status.cpu().numpy()


def test_device_tanh_vs_fp64():
    """The kernels' tanh (MUFU.EX2 + one MUFU.RCP per four values): absolute error against tanh in fp64."""
    from universal_differential_equations_b200 import _lib
    x = np.concatenate([np.linspace(-12, 12, 200001), np.random.default_rng(0).normal(0, 2, 200000), [0.0, 1e-8, -1e-8, 20.0, -20.0, 88.0, -88.0, 1e4, -1e4]]).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    yd = torch.empty_like(xd)
    rc = _lib.lib().b200ude_selftest_tanh(0, xd.data_ptr(), yd.data_ptr(), x.size, None)
    assert rc == 0
    torch.cuda.synchronize()
    err = np.abs(yd.cpu().numpy().astype(np.float64) - np.tanh(x.astype(np.float64)))
    rms, ymax = float(np.sqrt(np.mean(err ** 2))), float(np.abs(yd.cpu().numpy()).max())
    print(f"device tanh: max abs err {err.max():.3e}, rms {rms:.3e}, max |y| - 1 = {ymax - 1.0:.3e}")
    assert err.max() <= 6e-7, err.max()       # measured 4.8e-7 (near tanh = -1, where the error of 1/(1+e^2x) doubles)
    assert rms <= 2e-7, rms
    assert ymax <= 1.0 + 2.5e-7, ymax         # the batched inversion may overshoot +-1 by one or two ulp


def _family(monkeypatch, family, rows=0, groups=1):
    """Select the kernel family of the LV 2-32-32-2 chain: "wm" = warp-collective mma.sync (lv32_wm.cuh), "tc" = one trajectory per thread, 3xTF32 mma.sync sweeps
    through shared memory (lv32_tc.cuh), "auto" = the library's own choice; read by b200ude_create."""
    if family != "auto":
        monkeypatch.setenv("B200UDE_FWD_WM", "1" if family == "wm" else "0")
        monkeypatch.setenv("B200UDE_ADJ_WM", "1" if family == "wm" else "0")
    monkeypatch.setenv("B200UDE_WM_R", str(rows))
    monkeypatch.setenv("B200UDE_WM_G", str(groups))


@pytest.mark.parametrize("family", ["wm", "tc"])
@pytest.mark.parametrize("N", [1, 2, 31, 64, 65, 1000, 4097])
def test_lv32_forward_adjoint_vs_oracle(O, N, family, monkeypatch):
    _family(monkeypatch, family)
    ude = _ude()
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    m = O.lv_model()
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30, want_out=True)
    assert (status == 0).all()
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert abs(loss - l64) <= 1e-4 * abs(l64)
    assert np.linalg.norm(g - g64) <= 2e-3 * np.linalg.norm(g64)
    assert np.abs(gu - gu64).max() <= 2e-3 * np.abs(gu64).max()
    l32, g32, gu32 = O.ensemble_loss_grad(m, theta.astype(np.float32), u0, y, np.ones(2, np.float32), 0.1, 30)
    assert np.linalg.norm(g - g32) <= 2e-3 * np.linalg.norm(g64)
    solver.close()


@pytest.mark.parametrize("rows,groups,N", [(1, 1, 7), (1, 1, 8), (1, 1, 1001), (2, 1, 15), (2, 1, 16), (2, 2, 1001), (2, 2, 33)])
def test_lv32_warp_collective_variants_vs_oracle(O, rows, groups, N, monkeypatch):
    """The warp-collective family's launch variants: 8 or 16 trajectories per warp group, 1 or 2 groups per warp, ragged tails."""
    _family(monkeypatch, "wm", rows, groups)
    ude = _ude()
    theta = glorot_theta((2, 32, 32, 2), seed=4)
    u0, y = synthetic_ensemble(N, seed=3)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    m = O.lv_model()
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30, want_out=True)
    assert (status == 0).all()
    assert np.all(np.abs(out - out64) <= 1e-4 * (1 + np.abs(out64)))
    assert abs(loss - l64) <= 1e-5 * abs(l64)
    assert np.linalg.norm(g - g64) <= 2e-5 * np.linalg.norm(g64)      # measured 3e-7 ... 6e-7
    assert np.abs(gu - gu64).max() <= 2e-5 * np.abs(gu64).max()
    solver.close()


@pytest.mark.parametrize("fwd,adj", [("1", "0"), ("0", "1")])
def test_lv32_families_share_the_forward_record(O, fwd, adj, monkeypatch):
    """Either family's adjoint follows either family's forward (same ustep / dense layout)."""
    monkeypatch.setenv("B200UDE_FWD_WM", fwd)
    monkeypatch.setenv("B200UDE_ADJ_WM", adj)
    ude = _ude()
    N = 1000
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(O.lv_model(), theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30, want_out=True)
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert np.linalg.norm(g - g64) <= 1e-4 * np.linalg.norm(g64)
    assert np.abs(gu - gu64).max() <= 1e-4 * np.abs(gu64).max()
    solver.close()


@pytest.mark.parametrize("family", ["auto", "tc"])
def test_full_size_oracle_parity(O, family, monkeypatch):
    """The benchmarked size itself (N = 65 536, every SM loaded, several CTAs per SM): all trajectories,
    the loss, the full grad_theta and all of grad_u0 against the fp64 oracle."""
    _family(monkeypatch, family)
    ude = _ude()
    N = 65536
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(O.lv_model(), theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30, want_out=True)
    assert (status == 0).all()
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert abs(loss - l64) <= 1e-5 * abs(l64)
    assert np.linalg.norm(g - g64) <= 1e-4 * np.linalg.norm(g64)
    assert np.abs(g - g64).max() <= 1e-4 * np.abs(g64).max()
    assert np.abs(gu - gu64).max() <= 1e-4 * np.abs(gu64).max()
    solver.close()


def test_lv32_save_every_and_generic_cotangent(O):
    """dt = 0.05 with saveat = 0.1 (save_every = 2); generic dL/dout cotangent path == fused L2 path."""
    ude = _ude()
    N = 777
    theta = glorot_theta((2, 32, 32, 2), seed=3)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.05, 60, 2, max_trajectories=N)
    out, loss, g, gu, _ = _run(solver, theta, u0, y)
    m = O.lv_model()
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.05, 60, save_every=2, want_out=True)
    assert out.shape == (31, 2, N)
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert np.linalg.norm(g - g64) <= 2e-3 * np.linalg.norm(g64)
    cot = 2.0 * (torch.from_numpy(out).cuda() - torch.from_numpy(y).cuda())
    g2, gu2 = solver.adjoint(cot)
    torch.cuda.synchronize()
    assert np.linalg.norm(g2.cpu().numpy() - g) <= 1e-5 * np.linalg.norm(g)
    assert np.abs(gu2.cpu().numpy() - gu).max() <= 1e-5 * np.abs(gu).max()
    solver.close()


def test_lv32_deterministic_and_linear(O):
    """Bitwise run-to-run reproducibility; adjoint is linear in the cotangent; ensemble gradient is additive."""
    ude = _ude()
    N = 2048
    theta = glorot_theta((2, 32, 32, 2), seed=5)
    u0, y = synthetic_ensemble(N, seed=7)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out1, l1, g1, gu1, _ = _run(solver, theta, u0, y)
    out2, l2, g2, gu2, _ = _run(solver, theta, u0, y)
    assert np.array_equal(out1, out2) and np.array_equal(g1, g2) and np.array_equal(gu1, gu2) and l1 == l2
    cot = torch.randn(31, 2, N, device="cuda")
    ga, _ = solver.adjoint(cot)
    gb, _ = solver.adjoint(2.0 * cot)
    assert torch.allclose(gb, 2.0 * ga, rtol=1e-5, atol=1e-5 * float(ga.abs().max()))
    # additivity over a split of the ensemble
    h = N // 2
    _, la, gA, _, _ = _run(solver, theta, u0[:, :h].copy(), y[:, :, :h].copy(), want_gu0=False)
    _, lb, gB, _, _ = _run(solver, theta, u0[:, h:].copy(), y[:, :, h:].copy(), want_gu0=False)
    assert abs((la + lb) - l1) <= 1e-5 * abs(l1)
    assert np.linalg.norm(gA + gB - g1) <= 1e-4 * np.linalg.norm(g1)
    solver.close()


def test_lv32_host_buffer_entry_points(O):
    ude = _ude()
    N = 513
    theta = glorot_theta((2, 32, 32, 2), seed=2)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out, loss, g, gu, _ = _run(solver, theta, u0, y)
    out_h, status = solver.solve_host(theta, u0)
    assert np.array_equal(out_h, out) and (status == 0).all()
    gu_h = np.empty_like(u0)
    l_h, g_h, _ = solver.loss_gradient_host(theta, u0, y, grad_u0=gu_h)
    assert np.array_equal(g_h, g) and np.array_equal(gu_h, gu) and abs(l_h - loss) <= 1e-6 * abs(loss)
    solver.close()


def test_lv32_host_path_split_adjoint_is_bitwise_the_device_path():
    """Host-buffer call on a large ensemble: the data upload and the adjoint run in two halves of the trajectories (sub-range
    launches of the warp-collective adjoint); the partial rows, hence the sums, are those of the single launch."""
    ude = _ude()
    N = 20011
    theta = glorot_theta((2, 32, 32, 2), seed=5)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    _, loss, g, gu, _ = _run(solver, theta, u0, y)
    gu_h = np.empty_like(u0)
    l_h, g_h, _ = solver.loss_gradient_host(theta, u0, y, grad_u0=gu_h)
    assert np.array_equal(g_h, g) and np.array_equal(gu_h, gu) and abs(l_h - loss) <= 1e-6 * abs(loss)
    solver.close()


def test_autograd_concrete_solve_matches_adjoint(O):
    """loss.backward() through concrete_solve(EnsembleProblem) == fused adjoint == oracle."""
    ude = _ude()
    N = 300
    theta = glorot_theta((2, 32, 32, 2), seed=4)
    u0, y = synthetic_ensemble(N)
    f = _lv32(ude)
    prob = ude.EnsembleProblem(ude.ODEProblem(f, None, (0.0, 3.0), None), torch.from_numpy(u0).cuda())
    p = torch.from_numpy(theta).cuda().requires_grad_(True)
    pred = ude.concrete_solve(prob, ude.Tsit5(), p=p, saveat=0.1, dt=0.1, sensealg=ude.InterpolatingAdjoint(autojacvec=ude.ReverseDiffVJP()))
    loss = ((pred - torch.from_numpy(y).cuda()) ** 2).sum()
    loss.backward()
    m = O.lv_model()
    l64, g64, _ = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30)
    assert abs(float(loss.detach()) - l64) <= 1e-4 * abs(l64)
    assert np.linalg.norm(p.grad.cpu().numpy() - g64) <= 2e-3 * np.linalg.norm(g64)


@pytest.mark.parametrize("name,rates,acts,tend,nsub", [
    ("scenario_1", 0, ("rbf", "rbf", "rbf"), 3.0, 4),
    ("scenario_2", 1, ("rbf", "rbf", "rbf"), 6.0, 4),
    ("hudson_bay", 2, ("rbf", "rbf", "tanh"), 20.0, 8),
])
def test_reference_shapes_golden_forward(golden, O, name, rates, acts, tend, nsub):
    """KAT-2/5/8 on the GPU: the reference's trained parameters reproduce the reference's stored
    X-hat (its own Vern7@1e-6 solve) with the 2-5-5-5-2 kernels; tolerance = fp32 + the reference
    solver's own 1e-6..1e-5 error."""
    ude = _ude()
    g = golden[name]
    theta = g["theta_trained"].astype(np.float32)
    Xhat = g["Xhat"]
    n_save = Xhat.shape[1]
    save_dt = tend / (n_save - 1)
    f = _lv5(ude, acts, rates)
    solver = ude.UDESolver(f, 0.0, save_dt / nsub, (n_save - 1) * nsub, nsub, max_trajectories=4)
    u0 = np.repeat(g["X"][:, :1].astype(np.float32), 3, axis=1)
    out, status = solver.solve_host(theta, u0)
    assert (status == 0).all()
    scale = np.abs(Xhat).max()
    assert np.abs(out[:, :, 0].T - Xhat).max() <= 3e-4 * scale
    assert np.array_equal(out[:, :, 0], out[:, :, 2])
    solver.close()


@pytest.mark.parametrize("rates,acts", [(0, ("rbf", "rbf", "rbf")), (1, ("rbf", "rbf", "rbf")), (2, ("rbf", "rbf", "tanh"))])
def test_reference_shapes_adjoint_vs_oracle(golden, O, rates, acts):
    """2-5-5-5-2 chain with 0/1/2 trainable rates: gradient incl. the physics-rate entries vs the oracle."""
    ude = _ude()
    rng = np.random.default_rng(11)
    N = 193
    P = 87 + rates
    theta = (0.5 * rng.standard_normal(P)).astype(np.float32)
    if rates:
        theta[:rates] = rng.uniform(0.5, 1.5, rates)
    u0, y = synthetic_ensemble(N, n_steps=20, dt=0.05)
    f = _lv5(ude, acts, rates)
    solver = ude.UDESolver(f, 0.0, 0.05, 20, 1, max_trajectories=N)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    m = O.lv_model((2, 5, 5, 5, 2), acts + ("identity",), n_prefix=rates)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.05, 20, want_out=True)
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert abs(loss - l64) <= 1e-4 * abs(l64)
    assert np.linalg.norm(gth - g64) <= 2e-3 * np.linalg.norm(g64)
    if rates:
        assert np.all(np.abs(gth[:rates] - g64[:rates]) <= 2e-3 * np.abs(g64).max())
    assert np.abs(gu - gu64).max() <= 2e-3 * np.abs(gu64).max()
    solver.close()


def test_script_call_surface_seir_exposure(O):
    """SEIR_exposure/seir_exposure.jl:114-161 transcribed: ann / initial_params / ODEProblem / predict(theta) =
    concrete_solve(prob_nn, Vern7(), u0, theta, saveat, abstol, reltol, sensealg = InterpolatingAdjoint(autojacvec = ReverseDiffVJP()))
    / loss returning (l, pred) / callback(theta, l, pred) / sciml_train(ADAM) -> sciml_train(BFGS).  The only line that differs from
    the script is the one that builds prob_nn (it names the UDE form); the same dispatch is what julia/B200UDE.jl adds on the
    reference side."""
    ude = _ude()
    from universal_differential_equations_b200 import (ADAM, BFGS, FastChain, FastDense, InterpolatingAdjoint, ODEProblem, ReverseDiffVJP,
                                                        SEIRExposureUDE, Vern7, concrete_solve, initial_params, sciml_train)
    ann = FastChain(FastDense(3, 64, ude.tanh), FastDense(64, 64, ude.tanh), FastDense(64, 1))
    p = initial_params(ann, np.random.default_rng(0))
    p_ = O.SEIR_CONSTS
    u0 = np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0], np.float32)      # seir_exposure.jl:31-32 scale
    tspan, solution_t = (0.0, 21.0), np.arange(0.0, 22.0, 1.0)
    prob_nn = ODEProblem(SEIRExposureUDE(ann, p_), u0, tspan, p)                       # <- the changed line (seir_exposure.jl:131)
    noisy_data = torch.from_numpy(O.solve_fixed(O.seir_model(), np.zeros(len(p)), u0.astype(np.float64), 0.25, 84, save_every=4).T.astype(np.float32)).cuda()

    def predict(theta):
        # the script's call; tolerances 1e-4 instead of 1e-6 in the fp32 kernels (test_f64_seir_script_call_vern7_1e6 runs it
        # at the script's own Float64 / 1e-6)
        return concrete_solve(prob_nn, Vern7(), u0, theta, saveat=solution_t, abstol=1e-4, reltol=1e-4,
                              sensealg=InterpolatingAdjoint(autojacvec=ReverseDiffVJP()))

    def loss(theta):
        pred = predict(theta)
        return ((noisy_data[1:4, :] - pred[1:4, :]) ** 2).sum(), pred

    losses = []

    def callback(theta, l, pred):
        losses.append(l)
        assert pred.shape == (7, 22)
        return False

    res1 = sciml_train(loss, p, ADAM(0.01), cb=callback, maxiters=6)
    res2 = sciml_train(loss, res1.minimizer, BFGS(initial_stepnorm=0.01), cb=callback, maxiters=2)
    assert len(losses) >= 7 and np.isfinite(losses).all()
    assert res2.minimum <= losses[0]                       # training makes progress from the initial parameters
    assert float(loss(res2.minimizer)[0]) == pytest.approx(res2.minimum, rel=1e-3)


def test_script_call_surface_fisher_kpp(O):
    """FisherKPP/Fisher-KPP-CNN.jl:89-143,236-238 transcribed (26-point grid, reaction chain 1-10-20-10-1, theta = [p1; conv taps;
    conv bias; D0], predict_rd = concrete_solve(prob_nn, Tsit5(), rho0, theta, saveat = dt, sensealg = InterpolatingAdjoint(...)),
    loss with the |sum of the taps| penalty, sciml_train(ADAM))."""
    ude = _ude()
    from universal_differential_equations_b200 import (ADAM, FastChain, FastDense, FisherKPPUDE, InterpolatingAdjoint, ODEProblem,
                                                        ReverseDiffVJP, Tsit5, concrete_solve, initial_params, sciml_train)
    Nx, T, dt_save = 26, 5.0, 0.5
    X = 1.0
    dx = X / (Nx - 1)
    x = np.linspace(0.0, X, Nx)
    rho0 = (0.5 * (np.tanh((x - 0.4) / 0.02) - np.tanh((x - 0.6) / 0.02))).astype(np.float32)     # Fisher-KPP-CNN.jl:27-31 shape
    rx_nn = FastChain(FastDense(1, 10, ude.tanh), FastDense(10, 20, ude.tanh), FastDense(20, 10, ude.tanh), FastDense(10, 1))
    p1 = initial_params(rx_nn, np.random.default_rng(1))
    p = np.concatenate([p1, [1.1, -2.5, 1.0], [0.0], [6.5]]).astype(np.float32)      # init_w, conv bias, D0 (:100-108)
    prob_nn = ODEProblem(FisherKPPUDE(rx_nn, Nx), rho0, (0.0, T), p)                  # <- the changed line (:131)
    m = O.fkpp_model(Nx, (1, 10, 20, 10, 1), ("tanh", "tanh", "tanh", "identity"))
    ode_data = torch.from_numpy((0.9 * O.solve_fixed(m, p.astype(np.float64), rho0.astype(np.float64), 0.0125, 400, save_every=40).T).astype(np.float32)).cuda()

    def predict_rd(theta):
        return concrete_solve(prob_nn, Tsit5(), rho0, theta, saveat=dt_save, dt=0.0125,
                              sensealg=InterpolatingAdjoint(autojacvec=ReverseDiffVJP()))

    def loss_rd(theta):
        pred = predict_rd(theta)
        return ((ode_data - pred) ** 2).sum() + 10 ** 2 * theta[-5:-2].sum().abs(), pred     # :140-143

    losses = []
    res1 = sciml_train(loss_rd, p, ADAM(0.001), cb=lambda th, l, pred: (losses.append(l), False)[1], maxiters=8)
    assert len(losses) == 8 and np.isfinite(losses).all() and min(losses) < losses[0]
    assert res1.minimizer.shape == (len(p),)


# ---- double precision (dtype = B200UDE_F64): the precision the reference's LV scenario 1 / 2 and SEIR scripts run in ----
def _run64(solver, theta, u0, data, want_gu0=True):
    th = torch.from_numpy(np.asarray(theta, np.float64)).cuda()
    solver.set_params(th)
    status = torch.full((u0.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(np.asarray(u0, np.float64)).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(np.asarray(data, np.float64)).cuda(), want_grad_u0=want_gu0)
    torch.cuda.synchronize()
    return out.cpu().numpy(), float(loss), g.cpu().numpy(), (gu.cpu().numpy() if gu is not None else None), status.cpu().numpy()


@pytest.mark.parametrize("rates,acts", [(0, ("rbf", "rbf", "rbf")), (1, ("rbf", "rbf", "rbf")), (2, ("rbf", "rbf", "tanh"))])
def test_f64_lv_reference_shapes_vs_oracle(golden, O, rates, acts):
    """fp64 kernels, the reference's own LV shapes (scenario 1 / 2 / Hudson Bay: 2-5-5-5-2, 0 / 1 / 2 trainable rates), fixed-step
    Tsit5 + interpolating adjoint: the oracle is the same algorithm in C doubles -> agreement at round-off level."""
    ude = _ude()
    rng = np.random.default_rng(rates)
    N = 77
    f = _lv5(ude, acts, rates)
    P = 87 + rates
    theta = rng.normal(scale=0.3, size=P)
    if rates:
        theta[:rates] = rng.uniform(0.5, 2.0, rates)
    u0 = np.stack([rng.uniform(0.2, 1.0, N), rng.uniform(2.0, 5.0, N)])
    y = rng.normal(size=(31, 2, N))
    solver = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N, dtype=torch.float64)
    out, loss, g, gu, status = _run64(solver, theta, u0, y)
    m = O.lv_model((2, 5, 5, 5, 2), acts + ("identity",), n_prefix=rates)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta, u0, y, np.ones(2), 0.1, 30, want_out=True)
    assert (status == 0).all()
    assert np.abs(out - out64).max() <= 1e-11 * (1 + np.abs(out64).max())
    assert abs(loss - l64) <= 1e-11 * abs(l64)
    assert np.linalg.norm(g - g64) <= 1e-10 * np.linalg.norm(g64)
    assert np.abs(gu - gu64).max() <= 1e-10 * np.abs(gu64).max()
    # generic cotangent entry point
    cot = torch.from_numpy(2.0 * (out - y)).cuda()
    g2, gu2 = solver.adjoint(cot)
    assert np.linalg.norm(g2.cpu().numpy() - g) <= 1e-12 * np.linalg.norm(g)
    solver.close()


def test_f64_reference_call_scenario_1_vern7_1e6(golden, O):
    """The reference's own call in its own arithmetic: solve(prob, Vern7(); saveat = 0:0.05:3, abstol = reltol = 1e-6) in Float64
    (scenario_1.jl:41,84-85) from the stored start and trained parameters, against the reference's stored solution X-hat (KAT-2:
    the committed artefact was produced by exactly this call) and against the oracle; gradient (adaptive Tsit5 re-solve at the
    same tolerances) against the oracle's replay adjoint."""
    ude = _ude()
    g = golden["scenario_1"]
    f = _lv5(ude)
    theta = g["theta_trained"].astype(np.float64)
    N = 5
    u0 = np.repeat(g["X"][:, :1], N, axis=1).astype(np.float64)
    ts = np.linspace(0.0, 3.0, 61)
    solver = ude.UDESolver(f, 0.0, 0.05, 60, 1, max_trajectories=N, alg=ude.Vern7(), adaptive=True, abstol=1e-6, reltol=1e-6, max_steps=512,
                           dtype=torch.float64)
    rng = np.random.default_rng(0)
    y = rng.normal(size=(61, 2, N))
    out, loss, gth, gu, status = _run64(solver, theta, u0, y)
    assert (status == 0).all()
    assert np.abs(out[:, :, 0].T - g["Xhat"]).max() <= 2e-6          # the reference's own Vern7 @ 1e-6 solution (fp32 kernels: 3e-4)
    m = O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity"))
    o64, _, _ = O.solve_adaptive(m, theta, u0[:, 0], ts, 1e-6, 1e-6, solver=O.VERN7)
    assert np.abs(out[:, :, 0] - o64).max() <= 1e-7                  # same controller, same arithmetic up to libm's pow
    g_ref = np.zeros(87)
    for k in range(N):
        od, rec = O.solve_adaptive_dense(m, theta, u0[:, k], ts, 1e-6, 1e-6)
        gk, _ = O.adjoint_replay(m, theta, ts, rec, 2 * (od - y[:, :, k]))
        g_ref += gk
    assert np.linalg.norm(gth - g_ref) <= 1e-7 * np.linalg.norm(g_ref)
    solver.close()


def test_f64_seir_script_call_vern7_1e6(O):
    """seir_exposure.jl:137-141 in its own arithmetic: concrete_solve(prob_nn, Vern7(), u0, theta, saveat = 0:21, abstol = reltol =
    1e-6, sensealg = InterpolatingAdjoint(...)) in Float64 with populations of 1.4e7, against the oracle's Vern7 and, for the
    gradient, the oracle's replay adjoint of the adaptive Tsit5 solve."""
    ude = _ude()
    ann = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    p = ude.initial_params(ann, np.random.default_rng(0)).astype(np.float64)
    u0 = np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])[:, None]
    ts = np.arange(0.0, 22.0, 1.0)
    w = [0, 1, 1, 1, 0, 0, 0]
    solver = ude.UDESolver(ude.SEIRExposureUDE(ann), 0.0, 1.0, 21, 1, max_trajectories=1, alg=ude.Vern7(), adaptive=True, abstol=1e-6, reltol=1e-6,
                           max_steps=512, loss_weights=w, dtype=torch.float64)
    m = O.seir_model()
    data = O.solve_fixed(m, 0.9 * p, u0[:, 0], 0.25, 84, save_every=4)[:, :, None]
    out, loss, gth, gu, status = _run64(solver, p, u0, data)
    assert (status == 0).all()
    o64, _, _ = O.solve_adaptive(m, p, u0[:, 0], ts, 1e-6, 1e-6, solver=O.VERN7)
    scale = np.abs(o64).max(axis=0, keepdims=True) + 1.0
    assert np.all(np.abs(out[:, :, 0] - o64) <= 1e-9 * scale)
    od, rec = O.solve_adaptive_dense(m, p, u0[:, 0], ts, 1e-6, 1e-6)
    cot = 2 * np.asarray(w)[None, :] * (od - data[:, :, 0])
    g_ref, gu_ref = O.adjoint_replay(m, p, ts, rec, cot)
    assert np.linalg.norm(gth - g_ref) <= 1e-6 * np.linalg.norm(g_ref)
    assert np.abs(gu[:, 0] - gu_ref).max() <= 1e-6 * np.abs(gu_ref).max()
    solver.close()


def test_f64_adam_replays_reference_loss_history(golden):
    """KAT-4 on the GPU in the reference's arithmetic: sciml_train(loss, theta_init, ADAM(0.1)) with loss = sum(abs2, X - X-hat)
    (scenario_1.jl:91-94,114), predictions and gradients from the fp64 kernels (16 Tsit5 substeps per save interval), replays the
    stored losses[0..5] -- which pins the GPU gradient against the reference's own run."""
    ude = _ude()
    g = golden["scenario_1"]
    f = _lv5(ude)
    X = torch.from_numpy(g["X"].astype(np.float64)).cuda()
    prob = ude.ODEProblem(f, g["X"][:, 0].astype(np.float64), (0.0, 3.0), None)
    seen = []

    def loss(th):
        pred = ude.concrete_solve(prob, ude.Tsit5(), p=th, saveat=0.1, dt=0.1 / 16, sensealg=ude.InterpolatingAdjoint(), dtype=torch.float64)
        return ((X - pred) ** 2).sum()

    def cb(th, l):
        seen.append(l)
        return len(seen) >= 6
    th0 = torch.from_numpy(theta_scenario1_init(g)).cuda()
    ude.sciml_train(loss, th0, ude.ADAM(0.1), cb=cb, maxiters=10)
    ref = g["losses"][:6]
    assert np.all(np.abs(np.array(seen) - ref) <= 2e-6 * ref), (seen, ref)


def test_f64_unsupported_entry_points_fail_loudly():
    ude = _ude()
    from universal_differential_equations_b200 import _lib
    s = ude.UDESolver(_lv5(ude), 0.0, 0.1, 30, 1, max_trajectories=4, dtype=torch.float64)
    with pytest.raises(_lib.B200UDEError) as e:
        s.solve_host(np.zeros(87), np.ones((2, 4)))
    assert e.value.code == _lib.EUNSUPPORTED
    with pytest.raises(_lib.B200UDEError):
        s.adam_reset()
    with pytest.raises(_lib.B200UDEError):
        ude.UDESolver(ude.FisherKPPUDE(ude.FastChain(ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 1)), 26), 0.0, 0.01, 10, 1, dtype=torch.float64)
    s.close()


def test_error_behaviour():
    ude = _ude()
    from universal_differential_equations_b200._lib import B200UDEError, EINVAL, ESTATE, EUNSUPPORTED
    f = _lv32(ude)
    solver = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=64)
    with pytest.raises(B200UDEError) as e:
        solver.adjoint(torch.zeros(31, 2, 64, device="cuda"))
    assert e.value.code == ESTATE
    solver.set_params(torch.zeros(solver.P, device="cuda"))
    with pytest.raises(B200UDEError) as e:
        solver.forward(torch.zeros(2, 65, device="cuda"))
    assert e.value.code == EINVAL
    chain = ude.FastChain(ude.FastDense(2, 65, ude.tanh), ude.FastDense(65, 2))   # wider than any kernel supports
    with pytest.raises(B200UDEError) as e:
        ude.UDESolver(ude.LotkaVolterraUDE(chain), 0.0, 0.1, 30, 1, max_trajectories=8)
    assert e.value.code == EUNSUPPORTED
    # a diverging trajectory is flagged in status, the batch still completes
    theta = np.zeros(solver.P, np.float32)
    theta[-2:] = 3e38
    u0 = np.ones((2, 64), np.float32)
    _, status = solver.solve_host(theta, u0)
    assert (status == 1).all()
    solver.close()


def test_full_size_properties():
    """BASELINE size (65 536): permutation equivariance of the solve, invariance of the summed gradient."""
    ude = _ude()
    N = 65536
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    assert (status == 0).all() and np.isfinite(out).all() and np.isfinite(g).all()
    perm = np.random.default_rng(0).permutation(N)
    out_p, loss_p, g_p, gu_p, _ = _run(solver, theta, u0[:, perm].copy(), y[:, :, perm].copy())
    assert np.array_equal(out_p, out[:, :, perm]) and np.array_equal(gu_p, gu[:, perm])
    assert abs(loss_p - loss) <= 1e-5 * abs(loss)
    assert np.linalg.norm(g_p - g) <= 1e-4 * np.linalg.norm(g)
    solver.close()


def test_generic_lv_chain_vs_oracle(O):
    """A chain shape with no specialised kernel (2-16-16-2, tanh/rbf, one trainable rate) runs on the generic
    kernels and matches the oracle."""
    ude = _ude()
    rng = np.random.default_rng(5)
    N = 150
    chain = ude.FastChain(ude.FastDense(2, 16, ude.tanh), ude.FastDense(16, 16, ude.rbf), ude.FastDense(16, 2))
    f = ude.LotkaVolterraUDE(chain, trainable_rates=1)
    P = f.num_params()
    theta = (0.4 * rng.standard_normal(P)).astype(np.float32)
    theta[0] = 1.7
    u0, y = synthetic_ensemble(N, n_steps=20, dt=0.1)
    solver = ude.UDESolver(f, 0.0, 0.1, 20, 1, max_trajectories=N)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    m = O.lv_model((2, 16, 16, 2), ("tanh", "rbf", "identity"), n_prefix=1)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.1, 20, want_out=True)
    assert (status == 0).all()
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert abs(loss - l64) <= 1e-4 * abs(l64)
    assert np.linalg.norm(gth - g64) <= 2e-3 * np.linalg.norm(g64)
    assert np.abs(gu - gu64).max() <= 2e-3 * np.abs(gu64).max()
    # deterministic reduction: bitwise identical on a second run
    out2, loss2, gth2, gu2, _ = _run(solver, theta, u0, y)
    assert np.array_equal(gth, gth2) and loss == loss2
    solver.close()


def test_seir_exposure_ude_vs_oracle(O):
    """SEIR exposure UDE (7 states, chain 3-64-64-1 tanh on [S/N, I, D/N], seir_exposure.jl:114-130), Tsit5
    dt = 0.25 over (0, 21), saved daily, loss on rows E, I, R (seir_exposure.jl:146).  fp32 state with
    S, N ~ 1.4e7: per-component relative tolerances; adjoint parity for this model is oracle-only (unpinned)."""
    ude = _ude()
    rng = np.random.default_rng(9)
    N = 96
    chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    f = ude.SEIRExposureUDE(chain)
    theta = glorot_theta((3, 64, 64, 1), seed=2)
    S0 = 14e6
    u0 = np.zeros((7, N), np.float32)
    u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N)
    u0[1] = rng.uniform(0, 50, N); u0[2] = rng.uniform(0, 50, N); u0[3] = rng.uniform(0, 50, N)
    u0[4] = S0; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    n_steps, dt, every = 84, 0.25, 4
    m = O.seir_model()
    w = np.array([0, 1, 1, 1, 0, 0, 0], np.float64)
    # targets: the oracle's own solution for a perturbed theta (keeps residuals O(1))
    th2 = theta.astype(np.float64) * 1.05
    y = np.stack([O.solve_fixed(m, th2, u0[:, k].astype(np.float64), dt, n_steps, save_every=every) for k in range(N)], axis=2).astype(np.float32)
    solver = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=N, loss_weights=w)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, w, dt, n_steps, save_every=every, want_out=True)
    assert (status == 0).all() and out.shape == (22, 7, N)
    scale = np.abs(out64).max(axis=(0, 2), keepdims=True)
    assert np.all(np.abs(out - out64) <= 2e-5 * scale + 1e-3)
    # error budget of this configuration: the targets are the model's own solution for a 5 % perturbed theta, so the loss
    # cotangent 2 (u - y) is a difference of nearly equal fp32 numbers (residual rms 0.018 on states of 130: 4e-4 relative per
    # entry from fp32 storage alone); the fp32 ORACLE differs from the fp64 one by 3.6e-5 (loss) and 3.3e-5 (grad norm).
    l32, g32, _ = O.ensemble_loss_grad(m, theta.astype(np.float32), u0, y, w.astype(np.float32), dt, n_steps, save_every=every)
    e_l, e_g, e_g32 = abs(loss - l64) / abs(l64), np.linalg.norm(gth - g64) / np.linalg.norm(g64), np.linalg.norm(gth - g32) / np.linalg.norm(g64)
    print(f"SEIR: loss rel {e_l:.2e}, grad vs fp64 oracle {e_g:.2e}, vs fp32 oracle {e_g32:.2e} (fp32 oracle vs fp64: {np.linalg.norm(g32 - g64) / np.linalg.norm(g64):.2e})")
    assert e_l <= 5e-4       # measured 9.5e-5
    assert e_g <= 5e-4       # measured 6.8e-5 (round 1 allowed 1e-2 without a budget)
    assert e_g32 <= 3e-4     # measured 3.5e-5: against the fp32 oracle the kernels sit at the arithmetic's own noise
    solver.close()


@pytest.mark.parametrize("N", [1, 129, 300, 1000])
def test_seir_tensor_core_vs_runtime_shape_kernels(N, monkeypatch):
    """The tuned SEIR kernels (k_seir.cu: 3xTF32 mma.sync sweeps, two 128-trajectory groups per CTA) against the
    runtime-shape kernels (k_generic.cu) on ragged ensemble sizes, incl. a non-trivial cotangent path (adjoint with
    an explicit dL/dout) and grad_u0.  Both are fp32; they differ only in summation order / the 3xTF32 split."""
    ude = _ude()
    rng = np.random.default_rng(N)
    chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    f = ude.SEIRExposureUDE(chain)
    theta = glorot_theta((3, 64, 64, 1), seed=5)
    S0 = 14e6
    u0 = np.zeros((7, N), np.float32)
    u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N)
    u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = S0; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    y = rng.uniform(0, 100, (8, 7, N)).astype(np.float32)
    cot = rng.standard_normal((8, 7, N)).astype(np.float32)
    res = []
    for tc in ("1", "0"):
        monkeypatch.setenv("B200UDE_SEIR_TC", tc)
        solver = ude.UDESolver(f, 0.0, 0.25, 28, 4, max_trajectories=N, loss_weights=[0, 1, 1, 1, 0, 0, 0])
        out, loss, g, gu, status = _run(solver, theta, u0, y)
        g2, gu2 = solver.adjoint(torch.from_numpy(cot).cuda(), want_grad_u0=True)
        torch.cuda.synchronize()
        res.append((out, loss, g, gu, g2.cpu().numpy(), gu2.cpu().numpy()))
        assert (status == 0).all()
        rep = _run(solver, theta, u0, y)   # bitwise reproducible run to run
        assert np.array_equal(rep[0], out) and rep[1] == loss and np.array_equal(rep[2], g) and np.array_equal(rep[3], gu)
        solver.close()
    a, b = res
    scale = np.abs(b[0]).max(axis=(0, 2), keepdims=True)
    assert np.all(np.abs(a[0] - b[0]) <= 2e-6 * scale + 1e-4)
    assert abs(a[1] - b[1]) <= 1e-5 * abs(b[1])
    for k in (2, 3, 4, 5):
        assert np.linalg.norm(a[k] - b[k]) <= 2e-4 * np.linalg.norm(b[k]), k


@pytest.mark.parametrize("widths,acts,nx,N", [((1, 10, 20, 10, 1), ("tanh", "tanh", "tanh", "identity"), 26, 37),
                                             ((1, 5, 5, 5, 1), ("rbf", "rbf", "rbf", "identity"), 26, 5),
                                             ((1, 16, 16, 1), ("tanh", "tanh", "identity"), 256, 3)])
def test_fisher_kpp_upde_vs_oracle(O, widths, acts, nx, N):
    """Fisher-KPP UPDE (pointwise reaction chain + 3-tap periodic stencil, Fisher-KPP-CNN.jl:111-126): forward and
    interpolating adjoint incl. the stencil weights and D0 vs the oracle (parity for this model is oracle-only)."""
    ude = _ude()
    rng = np.random.default_rng(21)
    layers = [ude.FastDense(a, b, c) for a, b, c in zip(widths[:-1], widths[1:], acts)]
    f = ude.FisherKPPUDE(ude.FastChain(*layers), nx)
    m = O.fkpp_model(nx, widths, acts)
    P = O.num_params(m)
    assert P == f.num_params()
    theta = np.concatenate([glorot_theta(widths, seed=3), [1.1, -2.5, 1.0, 0.0, 6.5 if nx == 26 else 30.0]]).astype(np.float32)   # Fisher-KPP-CNN.jl:99-104
    x = np.linspace(0, 1, nx)
    u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) for d in rng.uniform(0.15, 0.5, N)], axis=1).astype(np.float32)
    n_steps, dt, every = 40, 0.0125 if nx == 26 else 0.002, 4
    y = (u0[None] * rng.uniform(0.8, 1.2, (n_steps // every + 1, 1, 1))).astype(np.float32)
    solver = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=N)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(nx), dt, n_steps, save_every=every, want_out=True)
    assert (status == 0).all() and out.shape == (n_steps // every + 1, nx, N)
    assert np.all(np.abs(out - out64) <= 3e-4 * (1 + np.abs(out64)))
    assert abs(loss - l64) <= 2e-4 * abs(l64)
    assert np.linalg.norm(gth - g64) <= 3e-3 * np.linalg.norm(g64)
    assert np.all(np.abs(gth[-5:] - g64[-5:]) <= 3e-3 * np.abs(g64[-5:]).max() + 1e-6)    # stencil weights, D0
    assert np.abs(gu - gu64).max() <= 3e-3 * np.abs(gu64).max()
    solver.close()


@pytest.mark.parametrize("nx,N", [(26, 7), (100, 3), (256, 5)])
def test_fisher_kpp_tuned_vs_runtime_shape_kernels(nx, N, monkeypatch):
    """Tuned 1-16-16-1 Fisher-KPP kernels (k_fkpp.cu) against the runtime-shape kernels: partially filled CTAs
    (7 trajectories at 4 per CTA), grids that are not a warp multiple, explicit cotangent and fused-L2 paths."""
    ude = _ude()
    rng = np.random.default_rng(nx)
    widths = (1, 16, 16, 1)
    layers = [ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)]
    f = ude.FisherKPPUDE(ude.FastChain(*layers), nx)
    theta = np.concatenate([glorot_theta(widths, seed=4), [1.1, -2.3, 0.9, 0.0, 0.01 * (nx - 1) ** 2]]).astype(np.float32)
    x = np.linspace(0, 1, nx)
    u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) for d in rng.uniform(0.15, 0.5, N)], axis=1).astype(np.float32)
    dt = 2.5 / (4 * 0.01 * (nx - 1) ** 2) / 4
    n_steps, every = 40, 8
    y = (np.repeat(u0[None], n_steps // every + 1, axis=0) + rng.normal(scale=0.05, size=(n_steps // every + 1, nx, N))).astype(np.float32)
    cot = rng.standard_normal(y.shape).astype(np.float32)
    res = []
    for tuned in ("1", "0"):
        monkeypatch.setenv("B200UDE_FKPP_TUNED", tuned)
        solver = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=N)
        out, loss, g, gu, status = _run(solver, theta, u0, y)
        g2, gu2 = solver.adjoint(torch.from_numpy(cot).cuda(), want_grad_u0=True)
        torch.cuda.synchronize()
        assert (status == 0).all()
        res.append((out, loss, g, gu, g2.cpu().numpy(), gu2.cpu().numpy()))
        rep = _run(solver, theta, u0, y)   # fixed-order reductions: bitwise reproducible run to run
        assert np.array_equal(rep[0], out) and rep[1] == loss and np.array_equal(rep[2], g) and np.array_equal(rep[3], gu)
        solver.close()
    a, b = res
    assert np.abs(a[0] - b[0]).max() <= 2e-6 * (1 + np.abs(b[0]).max())
    assert abs(a[1] - b[1]) <= 1e-5 * abs(b[1])
    for k in (2, 3, 4, 5):
        assert np.linalg.norm(a[k] - b[k]) <= 1e-4 * np.linalg.norm(b[k]), k


def test_fisher_kpp_golden_forward(golden, O):
    """KAT-6 on the GPU: scenario_3's trained parameters reproduce its stored X-hat (26 x 11, Float32)."""
    ude = _ude()
    g = golden["scenario_3"]
    chain = ude.FastChain(ude.FastDense(1, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 1))
    f = ude.FisherKPPUDE(chain, 26)
    solver = ude.UDESolver(f, 0.0, 0.5 / 40, 400, 40, max_trajectories=2)
    u0 = np.repeat(g["X"][:, :1].astype(np.float32), 2, axis=1)
    out, status = solver.solve_host(g["theta_trained"].astype(np.float32), u0)
    assert (status == 0).all()
    assert np.abs(out[:, :, 0].T - g["Xhat"]).max() <= 5e-4
    solver.close()


def test_adaptive_tsit5_forward_and_adjoint_vs_oracle(golden, O):
    """abstol / reltol path (scenario_1.jl:85: abstol = reltol = 1e-6): PI-controlled Tsit5 per trajectory with saveat by
    interpolation, and the interpolating adjoint replaying the accepted steps.  fp32 round-off can flip single
    accept/reject decisions, so values are compared, not step sequences; tolerances = a few x the solver tolerance."""
    ude = _ude()
    g = golden["scenario_1"]
    chain = ude.FastChain(ude.FastDense(2, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain)
    theta = g["theta_trained"].astype(np.float32)
    rng = np.random.default_rng(1)
    N = 70
    u0 = (g["X"][:, :1] * rng.uniform(0.8, 1.2, (2, N))).astype(np.float32)
    ts = np.linspace(0.0, 3.0, 31)
    tol = 1e-5
    m = O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity"))
    y = rng.normal(size=(31, 2, N)).astype(np.float32)
    solver = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=tol, reltol=tol, max_steps=256)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    assert (status == 0).all()
    l_ref, g_ref, gu_ref = 0.0, np.zeros(87), np.zeros((2, N))
    for k in range(N):
        o64, rec = O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol)
        assert np.abs(out[:, :, k] - o64).max() <= 50 * tol * (1 + np.abs(o64).max())
        dl = 2 * (o64 - y[:, :, k])
        l_ref += ((o64 - y[:, :, k]) ** 2).sum()
        gk, guk = O.adjoint_replay(m, theta.astype(np.float64), ts, rec, dl)
        g_ref += gk
        gu_ref[:, k] = guk
    assert abs(loss - l_ref) <= 1e-3 * abs(l_ref)
    assert np.linalg.norm(gth - g_ref) <= 5e-3 * np.linalg.norm(g_ref)
    assert np.abs(gu - gu_ref).max() <= 5e-3 * np.abs(gu_ref).max()
    # the golden X-hat of the reference (Vern7 @ 1e-6) is reproduced by the adaptive GPU solve from the reference's own start
    solver2 = ude.UDESolver(f, 0.0, 0.05, 60, 1, max_trajectories=2, adaptive=True, abstol=1e-6, reltol=1e-6, max_steps=512)
    o2, st2 = solver2.solve_host(theta, np.repeat(g["X"][:, :1].astype(np.float32), 2, axis=1))
    assert (st2 == 0).all() and np.abs(o2[:, :, 0].T - g["Xhat"]).max() <= 2e-4
    # step budget exhausted -> status 2, no crash
    solver3 = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=2, adaptive=True, abstol=1e-6, reltol=1e-6, max_steps=3)
    _, st3 = solver3.solve_host(theta, u0[:, :2].copy())
    assert (st3 == 2).all()
    for sv in (solver, solver2, solver3):
        sv.close()


@pytest.mark.parametrize("N,tol", [(300, 1e-5), (129, 1e-6)])
def test_adaptive_tensor_core_lv32_vs_oracle_and_runtime_shape(O, N, tol, monkeypatch):
    """Adaptive Tsit5 (abstol = reltol) on the tensor-core kernels of the headline chain: CTA-uniform attempt loops around
    the collective 32x32 sweeps, replay adjoint with the mma.sync gradient GEMM.  Against the fp64 oracle (values, not step
    sequences: fp32 round-off can flip accept/reject decisions) and against the runtime-shape adaptive kernels."""
    ude = _ude()
    rng = np.random.default_rng(N)
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, _ = synthetic_ensemble(N)
    y = rng.normal(size=(31, 2, N)).astype(np.float32)
    ts = np.linspace(0.0, 3.0, 31)
    res = {}
    for tc in ("1", "0"):
        monkeypatch.setenv("B200UDE_ADAPTIVE_TC", tc)
        solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=tol, reltol=tol, max_steps=256)
        res[tc] = _run(solver, theta, u0, y)
        assert (res[tc][4] == 0).all()
        solver.close()
    out, loss, gth, gu, _ = res["1"]
    m = O.lv_model()
    l_ref, g_ref, gu_ref = 0.0, np.zeros(1218), np.zeros((2, N))
    for k in range(N):
        o64, rec = O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol)
        assert np.abs(out[:, :, k] - o64).max() <= 50 * tol * (1 + np.abs(o64).max()) + 3e-5
        l_ref += ((o64 - y[:, :, k]) ** 2).sum()
        gk, guk = O.adjoint_replay(m, theta.astype(np.float64), ts, rec, 2 * (o64 - y[:, :, k]))
        g_ref += gk
        gu_ref[:, k] = guk
    assert abs(loss - l_ref) <= 1e-3 * abs(l_ref)
    assert np.linalg.norm(gth - g_ref) <= 5e-3 * np.linalg.norm(g_ref)
    assert np.abs(gu - gu_ref).max() <= 5e-3 * np.abs(gu_ref).max()
    o2, l2, g2, gu2, _ = res["0"]
    assert np.abs(out - o2).max() <= 50 * tol * (1 + np.abs(o2).max()) + 3e-5
    assert np.linalg.norm(gth - g2) <= 5e-3 * np.linalg.norm(g2)
    if N == 300:
        # step budget exhausted -> status 2 (no hang, no crash); the failure reaches the loss: the unreached save points are
        # NaN (as a failed retcode would signal), hence so is the gradient
        s3 = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=1e-7, reltol=1e-7, max_steps=3)
        o3, _, g3, _, st3 = _run(s3, theta, u0, y)
        assert (st3 == 2).all() and np.isnan(g3).all() and np.isnan(o3[-1]).all() and np.isfinite(o3[0]).all()
        # a diverging start -> status 1 for that trajectory only
        ub = u0.copy(); ub[:, 5] = 3e38
        s4 = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=tol, reltol=tol, max_steps=256)
        st4 = _run(s4, theta, ub, y)[4]
        assert st4[5] == 1 and (np.delete(st4, 5) == 0).all()
        s3.close(); s4.close()


def test_adaptive_tensor_core_seir_vs_oracle_and_runtime_shape(O, monkeypatch):
    """Adaptive Tsit5 on the SEIR exposure tensor-core kernels (seir_exposure.jl:137-141 style call: saveat daily over
    (0, 21), abstol = reltol): against the fp64 oracle (adaptive solve + replay adjoint) and the runtime-shape kernels.
    fp32 state with S, N ~ 1.4e7: per-component scales, tol = 1e-4."""
    ude = _ude()
    rng = np.random.default_rng(17)
    N, tol = 150, 1e-4
    chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    f = ude.SEIRExposureUDE(chain)
    theta = glorot_theta((3, 64, 64, 1), seed=2)
    S0 = 14e6
    u0 = np.zeros((7, N), np.float32)
    u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N)
    u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = S0; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    ts = np.linspace(0.0, 21.0, 22)
    m = O.seir_model()
    w = np.array([0, 1, 1, 1, 0, 0, 0], np.float64)
    ref = [O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol) for k in range(N)]
    y = (np.stack([r[0] for r in ref], axis=2) * (1 + 0.05 * rng.standard_normal((22, 7, N)))).astype(np.float32)
    res = {}
    for tc in ("1", "0"):
        monkeypatch.setenv("B200UDE_ADAPTIVE_TC", tc)
        solver = ude.UDESolver(f, 0.0, 1.0, 21, 1, max_trajectories=N, adaptive=True, abstol=tol, reltol=tol, max_steps=256, loss_weights=w)
        res[tc] = _run(solver, theta, u0, y)
        assert (res[tc][4] == 0).all()
        solver.close()
    out, loss, gth, gu, _ = res["1"]
    scale = np.abs(np.stack([r[0] for r in ref], axis=2)).max(axis=(0, 2), keepdims=True)
    l_ref, g_ref = 0.0, np.zeros(4481)
    for k in range(N):
        o64, rec = ref[k]
        assert np.all(np.abs(out[:, :, k] - o64) <= 50 * tol * scale[:, :, 0] + 1e-2)
        r = (o64 - y[:, :, k]) * w[None, :]
        l_ref += (w[None, :] * (o64 - y[:, :, k]) ** 2).sum()
        gk, _ = O.adjoint_replay(m, theta.astype(np.float64), ts, rec, 2 * r)
        g_ref += gk
    assert abs(loss - l_ref) <= 2e-2 * abs(l_ref)
    assert np.linalg.norm(gth - g_ref) <= 3e-2 * np.linalg.norm(g_ref)
    o2, l2, g2, gu2, _ = res["0"]
    assert np.all(np.abs(out - o2) <= 50 * tol * scale + 1e-2)
    assert np.linalg.norm(gth - g2) <= 3e-2 * np.linalg.norm(g2)


def test_vern7_fixed_step_forward_vs_oracle(golden, O):
    """solve(prob, Vern7(); saveat, adaptive=false): 9-stage 7th-order steps on the generic kernels vs the oracle's
    Vern7 (tableau = OrdinaryDiffEq's serialized constants, KAT-7).  The interpolating adjoint of a Vern7 handle runs
    over a Tsit5 re-solve with the same step (Vern7's dense output is not available): its gradient is compared with the
    oracle's Tsit5 interpolating adjoint."""
    ude = _ude()
    g = golden["scenario_1"]
    chain = ude.FastChain(ude.FastDense(2, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain)
    theta = g["theta_trained"].astype(np.float32)
    solver = ude.UDESolver(f, 0.0, 0.05, 60, 1, max_trajectories=8, alg=ude.Vern7())
    u0 = np.repeat(g["X"][:, :1].astype(np.float32), 5, axis=1)
    out, status = solver.solve_host(theta, u0)
    m = O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity"))
    ref = O.solve_fixed(m, g["theta_trained"], g["X"][:, 0], 0.05, 60, solver=O.VERN7)
    assert (status == 0).all()
    assert np.abs(out[:, :, 0] - ref).max() <= 2e-5 * (1 + np.abs(ref).max())
    assert np.abs(out[:, :, 0].T - g["Xhat"]).max() <= 2e-4      # the reference's own Vern7 solution
    # gradient through the Vern7 handle
    rng = np.random.default_rng(3)
    y = (out + rng.normal(scale=0.1, size=out.shape)).astype(np.float32)
    out2, loss, gth, gu, st = _run(solver, theta, u0, y)
    l64, g64, gu64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.05, 60)
    assert np.array_equal(out2, out)
    assert abs(loss - l64) <= 1e-4 * abs(l64)
    assert np.linalg.norm(gth - g64) <= 2e-3 * np.linalg.norm(g64)
    assert np.abs(gu - gu64).max() <= 2e-3 * np.abs(gu64).max()
    solver.close()


@pytest.mark.parametrize("tc", ["1", "0"])
def test_vern7_seir_tensor_core_forward_vs_oracle(O, tc, monkeypatch):
    """BASELINE config 3 as stated: the SEIR exposure UDE solved with Vern7 (seir_exposure.jl:138) -- fixed step on the tensor-core
    kernels (seir::vern7_forward_kernel) and, for comparison, on the runtime-shape kernels -- against the oracle's Vern7; the
    interpolating adjoint of the Vern7 handle (a Tsit5 re-solve on the same kernels) against the oracle's Tsit5 adjoint."""
    monkeypatch.setenv("B200UDE_SEIR_VERN7_TC", tc)
    ude = _ude()
    rng = np.random.default_rng(4)
    N = 300
    chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    theta = glorot_theta((3, 64, 64, 1), seed=2)
    S0 = 14e6
    u0 = np.zeros((7, N), np.float32)
    u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N)
    u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = S0; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    dt, n_steps, every = 0.5, 42, 2
    w = [0, 1, 1, 1, 0, 0, 0]
    solver = ude.UDESolver(ude.SEIRExposureUDE(chain), 0.0, dt, n_steps, every, max_trajectories=N, loss_weights=w, alg=ude.Vern7())
    y = rng.uniform(0, 100, (22, 7, N)).astype(np.float32)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    m = O.seir_model()
    assert (status == 0).all()
    for k in range(0, N, 37):
        ref = O.solve_fixed(m, theta.astype(np.float64), u0[:, k].astype(np.float64), dt, n_steps, solver=O.VERN7, save_every=every)
        scale = np.abs(ref).max(axis=0, keepdims=True)
        assert np.all(np.abs(out[:, :, k] - ref) <= 2e-5 * scale + 1e-3)
    l64, g64, gu64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.asarray(w, float), dt, n_steps, save_every=every)
    assert abs(loss - l64) <= 1e-3 * abs(l64)      # loss of the Tsit5 re-solve vs the oracle's Tsit5: same scheme
    assert np.linalg.norm(gth - g64) <= 1e-3 * np.linalg.norm(g64)
    solver.close()


def test_vern7_adaptive_forward_vs_oracle_and_reference(golden, O):
    """The reference's own call, solve(prob, Vern7(); saveat = 0:0.05:3, abstol = reltol = 1e-6) (scenario_1.jl:41,84-85),
    on the GPU: PI-controlled Vern7 with the save times as step end points (as the oracle's Vern7 path), from the reference's
    start and trained parameters, against the oracle and against the reference's stored X-hat; gradient via the adaptive
    Tsit5 re-solve."""
    ude = _ude()
    g = golden["scenario_1"]
    chain = ude.FastChain(ude.FastDense(2, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 5, ude.rbf), ude.FastDense(5, 2))
    f = ude.LotkaVolterraUDE(chain)
    theta = g["theta_trained"].astype(np.float32)
    rng = np.random.default_rng(5)
    N = 40
    u0 = (g["X"][:, :1] * rng.uniform(0.8, 1.2, (2, N))).astype(np.float32)
    u0[:, 0] = g["X"][:, 0]
    ts = np.linspace(0.0, 3.0, 61)
    tol = 1e-5
    m = O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity"))
    solver = ude.UDESolver(f, 0.0, 0.05, 60, 1, max_trajectories=N, alg=ude.Vern7(), adaptive=True, abstol=tol, reltol=tol, max_steps=512)
    y = rng.normal(size=(61, 2, N)).astype(np.float32)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    assert (status == 0).all()
    for k in range(0, N, 7):
        o64, _, _ = O.solve_adaptive(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol, solver=O.VERN7)
        assert np.abs(out[:, :, k] - o64).max() <= 50 * tol * (1 + np.abs(o64).max())
    assert np.abs(out[:, :, 0].T - g["Xhat"]).max() <= 3e-4
    # gradient: adaptive Tsit5 interpolating adjoint at the same tolerances
    l_ref, g_ref = 0.0, np.zeros(87)
    for k in range(N):
        o64, rec = O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol)
        l_ref += ((o64 - y[:, :, k]) ** 2).sum()
        gk, _ = O.adjoint_replay(m, theta.astype(np.float64), ts, rec, 2 * (o64 - y[:, :, k]))
        g_ref += gk
    assert abs(loss - l_ref) <= 1e-3 * abs(l_ref)
    assert np.linalg.norm(gth - g_ref) <= 5e-3 * np.linalg.norm(g_ref)
    solver.close()


@pytest.mark.parametrize("sens", ["interpolating", "forwarddiff"])
def test_on_device_adam_reproduces_reference_loss_history(golden, sens):
    """KAT-4 on the GPU: b200ude_train_adam (forward + adjoint + ADAM(0.1) without a host round trip, CUDA-graph
    replayed) from the reference's initial parameters reproduces the reference's stored loss history
    (scenario_1.jl:111-114; losses recorded at the pre-update theta).  fp32 state/gradient vs the reference's
    Float64 Vern7 + ForwardDiffSensitivity: 1e-4 relative on the first iterations, growing with the ADAM trajectory."""
    ude = _ude()
    g = golden["scenario_1"]
    theta0 = theta_scenario1_init(g).astype(np.float32)
    X = g["X"].astype(np.float32)                       # [2, 31]
    sub = 8
    # "forwarddiff": the sensealg the script itself uses (scenario_1.jl:86) = exact gradient of the discrete scheme
    solver = ude.UDESolver(_lv5(ude), 0.0, 0.1 / sub, 30 * sub, sub, max_trajectories=1,
                           sensealg=ude.ForwardDiffSensitivity() if sens == "forwarddiff" else ude.InterpolatingAdjoint())
    u0 = torch.from_numpy(np.ascontiguousarray(X[:, :1])).cuda()
    data = torch.from_numpy(np.ascontiguousarray(X.T[:, :, None])).cuda()   # [31, 2, 1]
    solver.set_params(torch.from_numpy(theta0).cuda())
    solver.adam_reset()
    losses = solver.train_adam(ude.ADAM(0.1), u0, data, 6).cpu().numpy()
    ref = g["losses"][:6]
    assert np.all(np.abs(losses[:3] - ref[:3]) <= 2e-4 * ref[:3]), (losses, ref)
    assert np.all(np.abs(losses - ref) <= 5e-3 * ref), (losses, ref)
    solver.close()


def test_on_device_adam_matches_host_driven_loop(monkeypatch):
    """b200ude_train_adam == the host-driven sciml_train loop over the same kernels (torch ADAM update), and the CUDA-graph
    replay == one-by-one launches bit for bit; L2 regularisation and loss scaling (scenario_2.jl:113-116) included."""
    ude = _ude()
    N, iters = 1000, 12
    theta0 = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    u0d, yd = torch.from_numpy(u0).cuda(), torch.from_numpy(y).cuda()
    scale, reg = 1.0 / N, 1e-3
    opt = ude.ADAM(0.01)
    hist = {}
    for graph in ("1", "0"):
        monkeypatch.setenv("B200UDE_TRAIN_GRAPH", graph)
        solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
        solver.set_params(torch.from_numpy(theta0).cuda())
        solver.adam_reset()
        l = solver.train_adam(opt, u0d, yd, iters, loss_scale=scale, l2_reg=reg).cpu().numpy()
        hist[graph] = (l, solver.get_params().cpu().numpy())
        solver.close()
    assert np.array_equal(hist["1"][0], hist["0"][0]) and np.array_equal(hist["1"][1], hist["0"][1])
    # host-driven: the same forward/adjoint through the device-pointer API, ADAM in torch
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    seen = []

    def loss(th):
        class F(torch.autograd.Function):
            @staticmethod
            def forward(ctx, t):
                solver.set_params(t)
                solver.forward(u0d)
                L, gth, _ = solver.adjoint_l2(yd)
                ctx.save_for_backward(gth, t)
                return scale * L[0] + reg * (t * t).sum()

            @staticmethod
            def backward(ctx, go):
                gth, t = ctx.saved_tensors
                return go * (scale * gth + 2 * reg * t)
        return F.apply(th)

    res = ude.sciml_train(loss, torch.from_numpy(theta0).cuda(), opt, cb=lambda th, l: seen.append(l) and False, maxiters=iters)
    seen = np.array(seen)
    assert np.all(np.abs(hist["1"][0] - seen) <= 1e-4 * np.abs(seen)), (hist["1"][0], seen)
    solver.close()
    # the chunked driver returns the same history
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    rec = []
    r = ude.sciml_train_l2(solver, theta0, u0d, yd, opt, cb=lambda th, l: rec.append(l) and False, maxiters=iters, chunk=5,
                           loss_scale=scale, l2_reg=reg)
    assert r.iterations == iters and np.array_equal(np.array(rec, np.float32), hist["1"][0])
    assert np.array_equal(r.final.cpu().numpy(), hist["1"][1])
    solver.close()


def test_peer_allreduce_single_rank_equals_plain_reduce():
    """The fused reduce + all-reduce kernel (NVLink peer-memory path, b200ude_adjoint_l2_allreduce) with world = 1 is the
    plain fixed-order reduce bit for bit, over repeated calls (epoch parity, monotonic flags).  The multi-rank exchange
    itself is exercised by tools/peer_allreduce_check.py under torchrun (needs >= 2 GPUs)."""
    ude = _ude()
    N = 3000
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    solver = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N)
    solver.set_params(torch.from_numpy(theta).cuda())
    u0d, yd = torch.from_numpy(u0).cuda(), torch.from_numpy(y).cuda()
    solver.forward(u0d)
    L0, g0, _ = solver.adjoint_l2(yd)
    L0, g0 = L0.clone(), g0.clone()
    pa = ude.PeerAllReduce(solver)
    for _ in range(5):
        L1, g1, gu = solver.adjoint_l2_allreduce(yd, want_grad_u0=True)
        torch.cuda.synchronize()
        assert torch.equal(L0, L1) and torch.equal(g0, g1)
    pa.close()
    solver.close()


@pytest.mark.parametrize("shape", ["lv32", "lv5", "lv5p2"])
def test_discrete_adjoint_forwarddiff_sensitivity_vs_oracle(O, shape):
    """sensealg = ForwardDiffSensitivity() (scenario_1.jl:86, hudson_bay.jl:102): the exact gradient of the discrete
    fixed-step Tsit5 scheme, computed by reverse accumulation through the stages (B200UDE_DISCRETE_ADJOINT), against the
    oracle's discrete adjoint (= torch autograd through the scheme to 1e-11, tests/test_oracle_golden.py) and, as a
    kernel-only check, against central finite differences of the GPU loss along a random direction."""
    ude = _ude()
    rng = np.random.default_rng(11)
    N = 200
    u0, y = synthetic_ensemble(N)
    if shape == "lv32":
        f, widths, acts, pre = _lv32(ude), (2, 32, 32, 2), ("tanh", "tanh", "identity"), 0
        theta = glorot_theta(widths, seed=1)
    else:
        rates = 2 if shape == "lv5p2" else 0
        f, widths, acts, pre = _lv5(ude, ("rbf", "rbf", "tanh"), rates), (2, 5, 5, 5, 2), ("rbf", "rbf", "tanh", "identity"), rates
        theta = np.concatenate([[1.3, 1.8][:rates], glorot_theta(widths, seed=2)]).astype(np.float32)
    m = O.lv_model(widths, acts, n_prefix=pre) if shape != "lv32" else O.lv_model()
    solver = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N, sensealg=ude.ForwardDiffSensitivity())
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    l64, g64, gu64 = O.ensemble_loss_grad_discrete(m, theta.astype(np.float64), u0.astype(np.float64), y.astype(np.float64), np.ones(2), 0.1, 30)
    assert (status == 0).all()
    assert abs(loss - l64) <= 1e-4 * abs(l64)
    assert np.linalg.norm(g - g64) <= 2e-4 * np.linalg.norm(g64)
    assert np.abs(gu - gu64).max() <= 2e-4 * np.abs(gu64).max()
    # the interpolating (continuous) adjoint differs from it by the truncation error only
    s2 = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N)
    _, _, gc, _, _ = _run(s2, theta, u0, y)
    assert 0 < np.linalg.norm(gc - g) <= 1e-3 * np.linalg.norm(g)
    # directional finite difference of the GPU loss itself (fp32: large step, loose tolerance)
    v = rng.standard_normal(theta.size).astype(np.float32)
    v /= np.linalg.norm(v)
    eps = 2e-2
    lp = _run(solver, theta + eps * v, u0, y)[1]
    lm = _run(solver, theta - eps * v, u0, y)[1]
    fd = (lp - lm) / (2 * eps)
    assert abs(fd - float(g @ v)) <= 2e-2 * abs(fd) + 1e-3 * np.linalg.norm(g)
    solver.close(); s2.close()


def test_discrete_adjoint_unsupported_configurations_fail_loudly():
    ude = _ude()
    from universal_differential_equations_b200._lib import B200UDEError, EUNSUPPORTED
    with pytest.raises(B200UDEError) as e:
        ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=4, sensealg=ude.ForwardDiffSensitivity(), adaptive=True, abstol=1e-6, reltol=1e-6)
    assert e.value.code == EUNSUPPORTED


def test_seir_neural_ode_baseline_vs_oracle(O):
    """dudt_node of the SEIR script (seir_exposure.jl:52-64; the black-box baseline trained before the UDE): chain
    7-64-64-64-7 tanh (P = 9287, the largest parameter vector of the path) on [S/N, E, I, R, N, D/N, C], five outputs used,
    dN and dC physical.  Runtime-shape kernels vs the oracle: forward, loss on E, I, R, gradient."""
    ude = _ude()
    rng = np.random.default_rng(23)
    N = 40
    widths = (7, 64, 64, 64, 7)
    chain = ude.FastChain(ude.FastDense(7, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 7))
    f = ude.SEIRNeuralODE(chain)
    assert f.num_params() == 9287
    theta = (0.3 * glorot_theta(widths, seed=6)).astype(np.float32)
    S0 = 14e6
    u0 = np.zeros((7, N), np.float32)
    u0[0] = 0.9 * S0 * rng.uniform(0.9, 1.0, N)
    u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = S0; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    n_steps, dt, every = 40, 0.25, 4
    m = O.seir_node_model()
    assert O.num_params(m) == 9287
    w = np.array([0, 1, 1, 1, 0, 0, 0], np.float64)
    y = np.stack([O.solve_fixed(m, theta.astype(np.float64) * 1.05, u0[:, k].astype(np.float64), dt, n_steps, save_every=every) for k in range(N)], axis=2).astype(np.float32)
    solver = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=N, loss_weights=w)
    out, loss, gth, gu, status = _run(solver, theta, u0, y)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, w, dt, n_steps, save_every=every, want_out=True)
    assert (status == 0).all()
    scale = np.abs(out64).max(axis=(0, 2), keepdims=True)
    assert np.all(np.abs(out - out64) <= 2e-5 * scale + 1e-3)
    assert abs(loss - l64) <= 5e-3 * abs(l64) + 1e-6
    assert np.linalg.norm(gth - g64) <= 1e-2 * np.linalg.norm(g64)
    solver.close()


def test_two_devices_in_one_process_interleaved():
    """One handle per device in ONE process, calls interleaved: constant tables, function attributes and launches follow
    the handle's device.  (Needs >= 2 GPUs; the benchmark itself runs one process per GPU.)"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    ude = _ude()
    N = 700
    theta = glorot_theta((2, 32, 32, 2), seed=1)
    u0, y = synthetic_ensemble(N)
    chain = ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))
    res = []
    solvers = [ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N, device=f"cuda:{d}") for d in (0, 1)]
    for rep in range(2):
        for d, sv in enumerate(solvers):
            with torch.cuda.device(d):
                dev = torch.device("cuda", d)
                sv.set_params(torch.from_numpy(theta).to(dev))
                out = sv.forward(torch.from_numpy(u0).to(dev))
                L, g, _ = sv.adjoint_l2(torch.from_numpy(y).to(dev))
                torch.cuda.synchronize(dev)
                res.append((out.cpu().numpy(), float(L), g.cpu().numpy()))
    for r in res[1:]:
        assert np.array_equal(r[0], res[0][0]) and r[1] == res[0][1] and np.array_equal(r[2], res[0][2])
    for sv in solvers:
        sv.close()


def test_peer_allreduce_two_ranks_vs_nccl():
    """Two ranks (one process per GPU, torchrun): the sums of the fused reduce + all-reduce over NVLink peer memory equal NCCL's
    all-reduce of the per-rank results and are bitwise identical on both ranks; the on-device multi-GPU ADAM loop keeps the
    replicas identical.  (Needs >= 2 GPUs; bench.py carries the same check in its JSON line for the 2/4/8-GPU runs.)"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29731", os.path.join(root, "tools", "peer_allreduce_check.py")], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "fused all-reduce OK" in r.stdout, r.stdout[-2000:]
    assert "replicas identical=True" in r.stdout, r.stdout[-2000:]


@pytest.mark.parametrize("nx,N,stages,dt,n_steps", [(64, 9, 6, 0.05, 20), (256, 3, 8, 0.0125, 16)])
def test_rkc2_stabilised_solver_fisher_kpp_vs_oracle(O, nx, N, stages, dt, n_steps):
    """solver = RKC2 (the closed-form ROCK2-class stabilised explicit method; ROCK2(eigen_est) in the reference's stiff PDE
    script, Climate/NeuralPDE/npde.jl:61) on the stiff Fisher-KPP grid at steps where Tsit5 is unstable (dt * rho = 8 / 33 vs
    its limit 3.3): forward solve, fused-L2 loss, interpolating adjoint (lambda stepped backwards by RKC2, cubic-Hermite dense
    output) against the oracle's RKC2 path, which converges with order 2 to the Tsit5 results (tests/test_oracle_golden.py)."""
    ude = _ude()
    rng = np.random.default_rng(nx)
    widths = (1, 16, 16, 1)
    layers = [ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)]
    f = ude.FisherKPPUDE(ude.FastChain(*layers), nx)
    D0 = 0.01 * (nx - 1) ** 2
    theta = np.concatenate([glorot_theta(widths, seed=3), [1.0, -2.0, 1.0, 0.0, D0]]).astype(np.float32)
    x = np.linspace(0, 1, nx)
    u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / 0.05) - np.tanh((x - (0.5 + d / 2)) / 0.05)) for d in rng.uniform(0.15, 0.5, N)], axis=1).astype(np.float32)
    every = n_steps // 4
    y = (0.9 * np.repeat(u0[None], 5, axis=0)).astype(np.float32)
    alg = ude.ROCK2(stages=stages)
    assert ude.ROCK2(eigen_est=4 * D0 + 2).n_stages(dt) <= stages        # the requested stage count covers dt * rho
    solver = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=N, alg=alg)
    out, loss, g, gu, status = _run(solver, theta, u0, y)
    assert (status == 0).all()
    m = O.fkpp_model(nx, widths, ("tanh", "tanh", "identity"))
    th64 = theta.astype(np.float64)
    l_ref, g_ref, gu_ref, o_ref = 0.0, np.zeros(theta.size), np.zeros((nx, N)), np.zeros((5, nx, N))
    for k in range(N):
        o, us, fs = O.solve_rkc2(m, th64, u0[:, k].astype(np.float64), dt, n_steps, stages, save_every=every, want_record=True)
        r = o - y[:, :, k]
        gk, guk = O.adjoint_rkc2(m, th64, us, fs, dt, n_steps, stages, 2 * r, save_every=every)
        l_ref += (r ** 2).sum(); g_ref += gk; gu_ref[:, k] = guk; o_ref[:, :, k] = o
    assert np.abs(out - o_ref).max() <= 1e-4 * (1 + np.abs(o_ref).max())
    assert abs(loss - l_ref) <= 1e-3 * abs(l_ref)
    assert np.linalg.norm(g - g_ref) <= 5e-3 * np.linalg.norm(g_ref)
    assert np.abs(gu - gu_ref).max() <= 5e-3 * np.abs(gu_ref).max()
    # Tsit5 at the same step is far outside its stability region
    s5 = ude.UDESolver(f, 0.0, dt, n_steps, every, max_trajectories=N)
    o5, st5 = s5.solve_host(theta, u0)
    assert (st5 != 0).any() or np.abs(o5).max() > 1e3
    solver.close(); s5.close()
