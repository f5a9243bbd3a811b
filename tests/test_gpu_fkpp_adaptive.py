"""Adaptive Tsit5 on the Fisher-KPP UPDE on the GPU (fkpp_adaptive.cuh), fp32 and fp64, forward and replay adjoint.

FisherKPP/Fisher-KPP-CNN.jl:136 trains through concrete_solve(prob_nn, Tsit5(), rho0, theta, saveat = dt, sensealg = ...) with
no dt: adaptive Tsit5 at OrdinaryDiffEq's default tolerances, in Float64.  The reference here is the oracle's adaptive solve with
the step record (solve_adaptive_dense) and its replay adjoint (adjoint_replay), per trajectory, in fp64.  fp32 round-off can flip
single accept / reject decisions, so the fp32 kernels are compared by value; the fp64 kernels take the oracle's step sequence.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import glorot_theta  # noqa: E402

TANH3 = ("tanh", "tanh", "tanh", "identity")
RBF3 = ("rbf", "rbf", "rbf", "identity")
TANH2 = ("tanh", "tanh", "identity")


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _chain(ude, widths, acts):
    return ude.FastChain(*[ude.FastDense(a, b, act) for a, b, act in zip(widths[:-1], widths[1:], acts)])


def _pulses(Nx, N, seed):
    """The script's initial pulse (Fisher-KPP-CNN.jl:27-31) with per-trajectory widths and heights: u0[Nx, N]."""
    rng = np.random.default_rng(seed)
    x = np.linspace(0.0, 1.0, Nx)
    half = rng.uniform(0.06, 0.2, N)
    amp = rng.uniform(0.8, 1.0, N)
    return (amp * 0.5 * (np.tanh((x[:, None] - 0.5 + half) / 0.02) - np.tanh((x[:, None] - 0.5 - half) / 0.02))).astype(np.float32)


def _theta(widths, taps, D0, seed=1):
    return np.concatenate([glorot_theta(widths, seed=seed), np.asarray(taps, np.float32), [0.0], [D0]]).astype(np.float32)


def _oracle_ref(O, m, theta, u0, ts, y, tol_abs, tol_rel, max_steps=4096):
    """Per trajectory: saved states, L2 loss, summed grad_theta, grad_u0 and accepted steps (fp64 oracle)."""
    th = theta.astype(np.float64)
    Nx, N = u0.shape
    out = np.empty((len(ts), Nx, N))
    g = np.zeros(len(theta))
    gu = np.empty((Nx, N))
    loss, nacc = 0.0, []
    for k in range(N):
        o, rec = O.solve_adaptive_dense(m, th, u0[:, k].astype(np.float64), ts, tol_abs, tol_rel, max_steps=max_steps)
        out[:, :, k] = o
        r = o - y[:, :, k]
        loss += (r ** 2).sum()
        gk, guk = O.adjoint_replay(m, th, ts, rec, 2.0 * r)
        g += gk
        gu[:, k] = guk
        nacc.append(rec[3])
    return out, loss, g, gu, nacc


def _check_fp32(out, loss, g, gu, ref, label, gu_bound=3e-3):
    o64, l64, g64, gu64 = ref[:4]
    assert np.abs(out - o64).max() <= 3e-4 * (1 + np.abs(o64)).max(), label
    assert abs(loss - l64) <= 1e-3 * abs(l64), label
    assert np.linalg.norm(g[:-5] - g64[:-5]) <= 3e-3 * np.linalg.norm(g64[:-5]), label                  # reaction chain
    sel = [-5, -4, -3, -1]                                                                              # w1, w2, w3, D0
    assert np.linalg.norm(g[sel] - g64[sel]) <= 3e-3 * np.linalg.norm(g64[sel]), label
    assert g[-2] == 0.0, label                                                                          # conv bias
    print(f"MEASURED fp32 {label} Nx={out.shape[1]} out={np.abs(out - o64).max():.2e} loss={abs(loss - l64) / abs(l64):.2e} "
          f"grad_theta={np.linalg.norm(g - g64) / np.linalg.norm(g64):.2e} grad_u0={np.abs(gu - gu64).max() / np.abs(gu64).max():.2e}")
    assert np.abs(gu - gu64).max() <= gu_bound * np.abs(gu64).max(), label


SHAPES = [  # Nx, widths, acts, N, T, taps, D0
    (26, (1, 10, 20, 10, 1), TANH3, 37, 5.0, (1.1, -2.5, 1.0), 6.5),      # the script's shape; 10 CTAs of 4, the last one partly filled
    (26, (1, 5, 5, 5, 1), RBF3, 5, 5.0, None, None),                        # scenario_3.jl's shape with its trained theta
    (100, (1, 16, 16, 1), TANH2, 3, 1.0, (1.0, -2.0, 1.0), 0.01 * 99 ** 2),
    (256, (1, 16, 16, 1), TANH2, 3, 0.5, (1.0, -2.0, 1.0), 0.01 * 255 ** 2),   # tuned fixed-step chain: routed to the runtime-shape kernels
]


@pytest.mark.parametrize("shape", SHAPES, ids=["script26_N37", "rbf26_N5", "grid100_N3", "grid256_N3"])
def test_fp32_vs_fp64_oracle(O, golden, shape):
    ude = _ude()
    Nx, widths, acts, N, T, taps, D0 = shape
    tol = 1e-5
    theta = golden["scenario_3"]["theta_trained"].astype(np.float32) if taps is None else _theta(widths, taps, D0)
    u0 = _pulses(Nx, N, seed=Nx + N)
    ts = np.linspace(0.0, T, 11)
    m = O.fkpp_model(Nx, widths, acts)
    # smooth data (0.9 x the solution, the script trains against a solution): rough data puts cotangent on the stiff grid modes,
    # which an explicit replay leaves undamped, so there grad_u0 depends on the exact step sequence (the fp32 and fp64 oracles
    # themselves differ by 2x on the 256-point grid with uniform-random data)
    y = (0.9 * _oracle_ref(O, m, theta, u0, ts, np.zeros((11, Nx, N)), tol, tol)[0]).astype(np.float32)
    ref = _oracle_ref(O, m, theta, u0, ts, y, tol, tol)
    solver = ude.UDESolver(ude.FisherKPPUDE(_chain(ude, widths, acts), Nx), 0.0, T / 10, 10, 1, max_trajectories=N, adaptive=True,
                           abstol=tol, reltol=tol, max_steps=1024)
    assert solver.P == len(theta)
    solver.set_params(torch.from_numpy(theta).cuda())
    status = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out_t = solver.forward(torch.from_numpy(u0).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)        # fused L2 (cotangent from the saved states)
    out = out_t.cpu().numpy()
    assert (status.cpu().numpy() == 0).all()
    gu_bound = 1e-2 if Nx == 256 else 3e-3   # fp32 vs fp64 oracle on the 256-point grid: 5.4e-3
    _check_fp32(out, float(loss), g.cpu().numpy(), gu.cpu().numpy(), ref, "l2", gu_bound)
    g2, gu2 = solver.adjoint(torch.from_numpy(2.0 * (out - y)).cuda())                         # explicit cotangent
    _check_fp32(out, float(((out.astype(np.float64) - y) ** 2).sum()), g2.cpu().numpy(), gu2.cpu().numpy(), ref, "cot", gu_bound)
    solver.close()


@pytest.mark.parametrize("abstol,reltol", [(1e-6, 1e-3), (1e-8, 1e-6)])
def test_fp64_vs_fp64_oracle(O, abstol, reltol):
    """fp64 kernels against the same algorithm in C doubles, the script's shape and tolerances."""
    ude = _ude()
    Nx, widths, N = 26, (1, 10, 20, 10, 1), 6
    theta = _theta(widths, (1.1, -2.5, 1.0), 6.5).astype(np.float64)
    u0 = _pulses(Nx, N, seed=3).astype(np.float64)
    ts = np.linspace(0.0, 5.0, 11)
    y = np.random.default_rng(4).uniform(0.0, 0.5, (11, Nx, N))
    m = O.fkpp_model(Nx, widths, TANH3)
    o64, l64, g64, gu64, nacc = _oracle_ref(O, m, theta, u0, ts, y, abstol, reltol)
    solver = ude.UDESolver(ude.FisherKPPUDE(_chain(ude, widths, TANH3), Nx), 0.0, 0.5, 10, 1, max_trajectories=N, adaptive=True,
                           abstol=abstol, reltol=reltol, max_steps=512, dtype=torch.float64)
    solver.set_params(torch.from_numpy(theta).cuda())
    status = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(u0).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)
    g2, gu2 = solver.adjoint(2.0 * (out - torch.from_numpy(y).cuda()))
    out, g, gu, g2, gu2 = (a.cpu().numpy() for a in (out, g, gu, g2, gu2))
    assert (status.cpu().numpy() == 0).all()
    e_out = np.abs(out - o64).max() / np.abs(o64).max()
    e_g = np.linalg.norm(g - g64) / np.linalg.norm(g64)
    e_gu = np.abs(gu - gu64).max() / np.abs(gu64).max()
    print(f"MEASURED fp64 fkpp adaptive tol=({abstol:g},{reltol:g}) steps={min(nacc)}-{max(nacc)} out={e_out:.2e} "
          f"loss={abs(float(loss) - l64) / l64:.2e} grad_theta={e_g:.2e} grad_u0={e_gu:.2e}")
    # (1e-6, 1e-3): the oracle's step sequence, round-off agreement.  (1e-8, 1e-6): round-off agreement up to t = 3, after which the
    # states separate by up to 3e-8 (measured on an H100), the size of abstol, as when one controller decision goes the other way;
    # the gradients still agree to 2e-10
    assert e_out <= max(1e-9, 5 * abstol)
    assert abs(float(loss) - l64) <= 1e-9 * l64
    assert e_g <= 1e-8 and e_gu <= 1e-8
    assert np.linalg.norm(g2 - g64) <= 1e-8 * np.linalg.norm(g64) and np.abs(gu2 - gu64).max() <= 1e-8 * np.abs(gu64).max()
    solver.close()


def test_script_call_surface_fisher_kpp_adaptive():
    """Fisher-KPP-CNN.jl:14-31, 55-66, 89-143, 236 transcribed with predict_rd exactly as the script writes it: no dt, so adaptive
    Tsit5 at abstol 1e-6 / reltol 1e-3.  Once in the mirror's default fp32 and once in Float64 (the script's precision)."""
    from scipy.integrate import solve_ivp
    ude = _ude()
    from universal_differential_equations_b200 import (ADAM, FastChain, FastDense, FisherKPPUDE, InterpolatingAdjoint, ODEProblem,
                                                        ReverseDiffVJP, Tsit5, concrete_solve, initial_params, sciml_train)
    D, r = 0.01, 1.0
    X, T = 1.0, 5.0
    dx, dt = 0.04, T / 10
    x = np.arange(0.0, X + dx / 2, dx)
    Nx = len(x)
    Amp, Delta = 1.0, 0.2
    rho0 = Amp * (np.tanh((x - (0.5 - Delta / 2)) / (Delta / 10)) - np.tanh((x - (0.5 + Delta / 2)) / (Delta / 10))) / 2
    lap = (np.diag(-2.0 * np.ones(Nx)) + np.diag(np.ones(Nx - 1), 1) + np.diag(np.ones(Nx - 1), -1)) / dx ** 2
    lap[0, -1] = lap[-1, 0] = 1.0 / dx ** 2

    def rc_ode(t, rho):
        return D * lap @ rho + r * rho * (1 - rho)
    sol = solve_ivp(rc_ode, (0.0, T), rho0, t_eval=np.linspace(0.0, T, 11), method="DOP853", rtol=1e-10, atol=1e-10)
    ode_data = sol.y   # Nx x 11

    rx_nn = FastChain(FastDense(1, 10, ude.tanh), FastDense(10, 20, ude.tanh), FastDense(20, 10, ude.tanh), FastDense(10, 1))
    p1 = initial_params(rx_nn, np.random.default_rng(1))
    p = np.concatenate([p1, [1.1, -2.5, 1.0], [0.0], [6.5]])
    prob_nn = ODEProblem(FisherKPPUDE(rx_nn, Nx), rho0, (0.0, T), p)

    histories = []
    for dtype in (torch.float32, torch.float64):
        data = torch.as_tensor(ode_data, dtype=dtype, device="cuda")
        kw = {} if dtype == torch.float32 else {"dtype": torch.float64}

        def predict_rd(theta):
            return concrete_solve(prob_nn, Tsit5(), rho0, theta, saveat=dt, sensealg=InterpolatingAdjoint(autojacvec=ReverseDiffVJP()), **kw)

        def loss_rd(theta):
            pred = predict_rd(theta)
            return ((data - pred) ** 2).sum() + 10 ** 2 * theta[-5:-2].sum().abs(), pred

        losses = []
        theta0 = p.astype(np.float32) if dtype == torch.float32 else torch.as_tensor(p, dtype=torch.float64, device="cuda")
        res = sciml_train(loss_rd, theta0, ADAM(0.001), cb=lambda th, l, pred: (losses.append(l), False)[1], maxiters=8)
        assert len(losses) == 8 and np.isfinite(losses).all() and min(losses) < losses[0], (dtype, losses)
        assert res.minimizer.shape == (len(p),) and res.minimizer.dtype == dtype
        histories.append(losses)
    assert abs(histories[0][0] - histories[1][0]) <= 1e-3 * histories[1][0], histories


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_kat6_scenario3_adaptive(golden, dtype):
    """KAT-6 with adaptive Tsit5: scenario_3's trained parameters from X[:, 1] reproduce its stored X-hat (Vern7, Float32)."""
    ude = _ude()
    g = golden["scenario_3"]
    f = ude.FisherKPPUDE(_chain(ude, (1, 5, 5, 5, 1), RBF3), 26)
    solver = ude.UDESolver(f, 0.0, 0.5, 10, 1, max_trajectories=2, adaptive=True, abstol=1e-7, reltol=1e-5, max_steps=512, dtype=dtype)
    u0 = np.repeat(g["X"][:, :1], 2, axis=1)
    if dtype == torch.float32:
        out, status = solver.solve_host(g["theta_trained"].astype(np.float32), u0.astype(np.float32))
    else:
        solver.set_params(torch.from_numpy(g["theta_trained"].astype(np.float64)).cuda())
        st = torch.full((2,), -1, dtype=torch.int32, device="cuda")
        out = solver.forward(torch.from_numpy(u0.astype(np.float64)).cuda(), status=st).cpu().numpy()
        status = st.cpu().numpy()
    assert (status == 0).all()
    assert np.abs(out[:, :, 0].T - g["Xhat"]).max() <= 2e-4
    assert np.array_equal(out[:, :, 0], out[:, :, 1])
    solver.close()


def _script_solver(ude, N, dtype=torch.float32, max_steps=512):
    f = ude.FisherKPPUDE(_chain(ude, (1, 10, 20, 10, 1), TANH3), 26)
    return ude.UDESolver(f, 0.0, 0.5, 10, 1, max_trajectories=N, adaptive=True, max_steps=max_steps, dtype=dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_max_steps_status_and_nan(dtype):
    ude = _ude()
    N = 5
    solver = _script_solver(ude, N, dtype, max_steps=3)
    solver.set_params(torch.from_numpy(_theta((1, 10, 20, 10, 1), (1.1, -2.5, 1.0), 6.5)).to("cuda", dtype))
    st = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(_pulses(26, N, seed=5)).to("cuda", dtype), status=st).cpu().numpy()
    assert (st.cpu().numpy() == 2).all()
    assert np.isfinite(out[0]).all()
    for k in range(N):
        assert np.isnan(out[-1, :, k]).all(), k
    solver.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
def test_trajectory_isolation_and_determinism(O, dtype):
    """Trajectories that need different step counts share CTAs: each one's saved states, status and grad_u0 are bitwise those of
    the same trajectory solved alone (finished trajectories idle without recording; the norm is summed in point order), and two
    runs are bitwise identical, grad_theta and loss included."""
    ude = _ude()
    N = 9   # three CTAs of four trajectories, the last one partly filled
    theta = _theta((1, 10, 20, 10, 1), (1.1, -2.5, 1.0), 6.5)
    u0 = _pulses(26, N, seed=7)
    y = np.random.default_rng(8).uniform(0.0, 0.5, (11, 26, N))
    cot = np.random.default_rng(9).normal(size=(11, 26, N))
    m = O.fkpp_model(26, (1, 10, 20, 10, 1), TANH3)
    steps = {O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), np.linspace(0, 5, 11), 1e-6, 1e-3)[1][3]
             for k in range(N)}
    assert len(steps) > 1, steps
    solver = _script_solver(ude, N, dtype)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)  # noqa: E731
    solver.set_params(dev(theta))

    def run(sl):
        st = torch.full((sl.stop - sl.start,), -1, dtype=torch.int32, device="cuda")
        out = solver.forward(dev(u0[:, sl]), status=st)
        g, gu = solver.adjoint(dev(cot[:, :, sl]))
        loss, gl, gul = solver.adjoint_l2(dev(y[:, :, sl]), want_grad_u0=True)
        return [a.cpu().numpy() for a in (out, st, g, gu, loss, gl, gul)]

    full = run(slice(0, N))
    assert (full[1] == 0).all()
    again = run(slice(0, N))
    for a, b in zip(full, again):
        assert np.array_equal(a, b)
    for k in range(N):
        one = run(slice(k, k + 1))
        assert np.array_equal(one[0][:, :, 0], full[0][:, :, k]), k
        assert one[1][0] == full[1][k], k
        assert np.array_equal(one[3][:, 0], full[3][:, k]), k
        assert np.array_equal(one[6][:, 0], full[6][:, k]), k
    solver.close()


def test_host_buffer_entry_points_and_train_adam():
    """The host-buffer pair (what the Julia shim calls) is bitwise the device-pointer path; train_adam is bitwise the same
    iterations launched one by one."""
    ude = _ude()
    N = 6
    theta = _theta((1, 10, 20, 10, 1), (1.1, -2.5, 1.0), 6.5)
    u0 = _pulses(26, N, seed=11)
    y = np.random.default_rng(12).uniform(0.0, 0.5, (11, 26, N)).astype(np.float32)
    solver = _script_solver(ude, N)
    solver.set_params(torch.from_numpy(theta).cuda())
    st = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(u0).cuda(), status=st)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(y).cuda(), want_grad_u0=True)
    out_h, st_h = solver.solve_host(theta, u0)
    assert np.array_equal(out_h, out.cpu().numpy()) and np.array_equal(st_h, st.cpu().numpy())
    gu_h = np.empty((26, N), np.float32)
    l_h, g_h, _ = solver.loss_gradient_host(theta, u0, y, grad_u0=gu_h)
    assert np.float32(l_h) == float(loss) and np.array_equal(g_h, g.cpu().numpy()) and np.array_equal(gu_h, gu.cpu().numpy())

    opt = ude.ADAM(0.001)
    iters = 4
    solver.set_params(torch.from_numpy(theta).cuda())
    solver.adam_reset()
    hist = solver.train_adam(opt, torch.from_numpy(u0).cuda(), torch.from_numpy(y).cuda(), iters).cpu().numpy()
    th_graph = solver.get_params().cpu().numpy()
    solver.set_params(torch.from_numpy(theta).cuda())
    solver.adam_reset()
    ref = []
    for _ in range(iters):
        out_i = solver.forward(torch.from_numpy(u0).cuda())   # noqa: F841  (the fused L2 of an adaptive solve reads it)
        l, gi, _ = solver.adjoint_l2(torch.from_numpy(y).cuda())
        ref.append(float(l))
        solver.adam_step(opt, gi)
    torch.cuda.synchronize()
    assert np.isfinite(hist).all() and hist[0] == float(loss)
    assert np.array_equal(hist, np.asarray(ref, np.float32))
    assert np.array_equal(th_graph, solver.get_params().cpu().numpy())
    solver.close()
