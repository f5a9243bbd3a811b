"""The checkpointed record of adaptive Tsit5 on the Fisher-KPP UPDE (B200UDE_FLAG_CHECKPOINT, InterpolatingAdjoint(checkpointing =
true)) on the GPU, fp32 and fp64.

The forward keeps u_n every K = max(1, round(sqrt(max_steps / 7))) accepted steps and the step sizes; the adjoint recomputes each
segment of K steps with the forward's own stage code and replays it.  Everything is compared bitwise with the full record (the same
inputs on a handle without the flag): saved states, status, loss, grad_theta and grad_u0.  The accepted step counts are not exposed;
the replay adjoint reads them and the step times, so they are covered by the adjoint's bitwise agreement.
"""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import glorot_theta  # noqa: E402

RBF = ((1, 5, 5, 5, 1), ("rbf", "rbf", "rbf", "identity"))
TANH = ((1, 16, 16, 1), ("tanh", "tanh", "identity"))
# Nx -> (T, candidate D0): stiff enough that the steps are limited by stability, so that the step counts of the pulses sit close
# together far above those of the flat states (a few steps); the first D0 whose ensemble has every category below is used
GRIDS = {3: (5.0, (300.0, 320.0)), 26: (5.0, (70.0, 75.0, 80.0)), 100: (0.5, (0.01 * 99 ** 2, 100.0)), 256: (0.2, (0.01 * 255 ** 2, 660.0))}


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _seg(max_steps):
    return max(1, math.floor(math.sqrt(max_steps / 7) + 0.5))


def _chain(ude, widths, acts):
    return ude.FastChain(*[ude.FastDense(a, b, act) for a, b, act in zip(widths[:-1], widths[1:], acts)])


def _theta(widths, D0, taps=(1.0, -2.0, 1.0)):
    return np.concatenate([glorot_theta(widths, seed=1), np.asarray(taps, np.float32), [0.0], [D0]]).astype(np.float32)


def _u0s(Nx):
    """Flat states (a few steps), pulses and noise of several sizes (steps close to the stability limit): u0[Nx, n]."""
    x = np.linspace(0, 1, Nx)
    rng = np.random.default_rng(Nx)
    g = lambda c, w: np.exp(-((x - c) / w) ** 2)  # noqa: E731
    alt = (-1.0) ** np.arange(Nx)
    cols = [np.full(Nx, 0.3), rng.uniform(0, 1, Nx), 0.5 + 0.5 * np.sin(2 * np.pi * x), 5 * g(.5, .1), np.zeros(Nx),
            rng.uniform(0, .1, Nx), -g(.4, .1), 0.5 + 0.1 * alt, 0.01 * g(.5, .1), 0.5 + 0.5 * np.sin(8 * np.pi * x), 0.5 + 0.01 * alt]
    cols += [a * rng.uniform(0, 1, Nx) for a in (0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.2, 1.5)] + [0.8 * g(0.3, w) for w in (0.05, 0.2)]
    return np.stack(cols, axis=1).astype(np.float32)


def _pick(S):
    """max_steps (and K) under which the ensemble has trajectories with nacc < K, nacc a multiple of K, nacc > K not a multiple
    of K, and at least one that runs out of steps (the margin of 3 keeps that so in fp32, whose step counts may differ by one)."""
    for M in range(max(S) - 3, 7, -1):
        K = _seg(M)
        ok = [s for s in S if s <= M]
        if any(s > M for s in S) and any(s < K for s in ok) and any(s % K == 0 and s >= K for s in ok) and any(s % K and s > K for s in ok):
            return M, K
    return None


def _case(O, Nx, chain):
    widths, acts = chain
    T, D0s = GRIDS[Nx]
    m = O.fkpp_model(Nx, widths, acts)
    u0 = _u0s(Nx)
    ts = np.linspace(0.0, T, 11)
    for D0 in D0s:
        theta = _theta(widths, D0)
        S = [O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, 1e-6, 1e-3, max_steps=100000)[1][3]
             for k in range(u0.shape[1])]
        sel = _pick(S)
        if sel:
            return theta, u0, T, sel[0], sel[1], S
    raise AssertionError(f"no max_steps gives every step-count category on {Nx} points")


def _blowup(Nx, dtype):
    """A finite state whose first right-hand side overflows: the solve stops at once with status 1 (nacc = 0)."""
    big = 3e38 if dtype == torch.float32 else 1e308
    return big * (-1.0) ** np.arange(Nx)


def _solver(ude, chain, Nx, T, N, M, dtype, ckpt):
    return ude.UDESolver(ude.FisherKPPUDE(_chain(ude, *chain), Nx), 0.0, T / 10, 10, 1, max_trajectories=N, adaptive=True, abstol=1e-6,
                         reltol=1e-3, max_steps=M, dtype=dtype, sensealg=ude.InterpolatingAdjoint(checkpointing=ckpt))


def _run(solver, theta, u0, cot, y, dtype):
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)  # noqa: E731
    N = u0.shape[1]
    solver.set_params(dev(theta))
    st = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(dev(u0), status=st)
    g, gu = solver.adjoint(dev(cot))
    loss, gl, gul = solver.adjoint_l2(dev(y), want_grad_u0=True)
    return [a.cpu().numpy() for a in (out, st, g, gu, loss, gl, gul)]


NAMES = ("out", "status", "grad_theta(cot)", "grad_u0(cot)", "loss(l2)", "grad_theta(l2)", "grad_u0(l2)")


def _same(a, b, label):
    for name, x, y in zip(NAMES, a, b):
        assert x.dtype == y.dtype and x.shape == y.shape, (label, name)
        assert np.array_equal(x, y, equal_nan=True), (label, name, np.nanmax(np.abs(x.astype(np.float64) - y)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("Nx", [3, 26, 100, 256])
@pytest.mark.parametrize("chain", [RBF, TANH], ids=["rbf_1-5-5-5-1", "tanh_1-16-16-1"])
def test_bitwise_flag_on_vs_off(O, dtype, Nx, chain):
    ude = _ude()
    theta, u0, T, M, K, S = _case(O, Nx, chain)
    # one trajectory that goes non-finite, among the first ones so that it shares a CTA with others on the small grids
    u0 = np.insert(u0, 2, _blowup(Nx, dtype), axis=1)
    N = u0.shape[1]
    rng = np.random.default_rng(Nx)   # cotangent and data uniform in space: a rough cotangent excites the stiff grid modes
    cot = np.repeat(rng.normal(size=(11, 1, N)), Nx, axis=1)
    y = np.repeat(rng.uniform(0.0, 0.5, (11, 1, N)), Nx, axis=1)
    # the sub-ensemble of stability-limited solves that end well inside max_steps (fp32 step counts may differ from the fp64
    # oracle's by a step or two): no NaN reaches its loss or gradients.  The flat states are left out of it: their few steps are far
    # beyond the stencil's stability limit, and the replay over them can leave the fp32 range
    clean = [k + (k >= 2) for k in range(len(S)) if 20 < S[k] <= M - 5]
    res = {}
    for ckpt in (False, True):
        s = _solver(ude, chain, Nx, T, N, M, dtype, ckpt)
        full = _run(s, theta, u0, cot, y, dtype)
        part = _run(s, theta, u0[:, clean], cot[:, :, clean], y[:, :, clean], dtype)
        res[ckpt] = (full, part)
        s.close()
    (full0, clean0), (full1, clean1) = res[False], res[True]
    st = full1[1]
    print(f"MEASURED checkpoint {dtype} Nx={Nx} K={K} max_steps={M} oracle steps={sorted(S)} status={st.tolist()}")
    assert st[2] == 1 and (st == 2).any() and (st == 0).any(), st
    assert (clean1[1] == 0).all() and all(np.isfinite(a).all() for a in clean1[2:])
    ok = np.flatnonzero(st == 0)
    assert np.isfinite(full1[3][:, ok]).all() and np.isfinite(full1[6][:, ok]).all()
    _same(full0, full1, "with the non-finite trajectory")
    _same(clean0, clean1, "the trajectories that finish")


def _device_bytes(solver):
    return int(solver._L.b200ude_device_bytes(solver._h))


def test_capacity_256_points_8192_trajectories(O):
    """max_steps = 2048 on 256 points: the full record of 8192 trajectories (~120 GB) does not fit on the card, the checkpointed one
    (~2 GB) does; sampled trajectories are bitwise those solved alone, with and without the flag."""
    from universal_differential_equations_b200 import _lib
    ude = _ude()
    Nx, N, M, T = 256, 8192, 2048, 0.2
    K = _seg(M)
    assert K == 17
    theta = _theta(TANH[0], 0.01 * 255 ** 2)
    P = len(theta)
    with pytest.raises(_lib.B200UDEError) as e:
        _solver(ude, TANH, Nx, T, N, M, torch.float32, False)
    assert e.value.code == _lib.ENOMEM
    s = _solver(ude, TANH, Nx, T, N, M, torch.float32, True)
    # the documented record: theta (float4-padded), checkpoints, scratch, partial rows (8 warps per 256-point CTA), grad, loss,
    # step times, nacc, the L2 cotangent, step sizes, per-block losses
    n_save = 11
    reals = (((P + 3) // 4) * 4 + ((M + K - 1) // K + 1) * Nx * N + (7 * K + 2) * Nx * N + 8 * N * (P + 1) + P + 1 + (M + 1) * N
             + n_save * Nx * N + M * N + 296)
    assert _device_bytes(s) == 4 * reals + 4 * N
    print(f"MEASURED checkpoint capacity device_bytes={_device_bytes(s)} (full record would be "
          f"{4 * ((M + 1 + 6 * M + 1) * Nx * N)} B of ustep + dense alone)")
    rng = np.random.default_rng(5)
    x = np.linspace(0.0, 1.0, Nx)
    half, amp = rng.uniform(0.06, 0.2, N), rng.uniform(0.3, 1.0, N)
    u0 = (amp * 0.5 * (np.tanh((x[:, None] - 0.5 + half) / 0.02) - np.tanh((x[:, None] - 0.5 - half) / 0.02))).astype(np.float32)
    cot = rng.normal(size=(n_save, Nx, N)).astype(np.float32)
    y = rng.uniform(0.0, 0.5, (n_save, Nx, N)).astype(np.float32)
    full = _run(s, theta, u0, cot, y, torch.float32)
    s.close()
    assert (full[1] == 0).all() and np.isfinite(full[2]).all() and np.isfinite(full[5]).all()
    pick = rng.choice(N, 8, replace=False)
    for ckpt in (False, True):
        one = _solver(ude, TANH, Nx, T, 1, M, torch.float32, ckpt)
        for k in pick:
            r = _run(one, theta, u0[:, k:k + 1], cot[:, :, k:k + 1], y[:, :, k:k + 1], torch.float32)
            assert np.array_equal(r[0][:, :, 0], full[0][:, :, k]) and r[1][0] == full[1][k], (ckpt, k)
            assert np.array_equal(r[3][:, 0], full[3][:, k]) and np.array_equal(r[6][:, 0], full[6][:, k]), (ckpt, k)
        one.close()


def test_train_adam_and_host_buffers():
    """train_adam (one CUDA graph per call) and the host-buffer entry points give bitwise the theta, losses and outputs of a handle
    without the flag; two runs are bitwise identical."""
    ude = _ude()
    widths, acts = (1, 10, 20, 10, 1), ("tanh", "tanh", "tanh", "identity")
    Nx, N = 26, 6
    theta = _theta(widths, 6.5, (1.1, -2.5, 1.0))
    rng = np.random.default_rng(11)
    x = np.linspace(0.0, 1.0, Nx)
    half = rng.uniform(0.06, 0.2, N)
    u0 = (0.5 * (np.tanh((x[:, None] - 0.5 + half) / 0.02) - np.tanh((x[:, None] - 0.5 - half) / 0.02))).astype(np.float32)
    y = rng.uniform(0.0, 0.5, (11, Nx, N)).astype(np.float32)
    opt = ude.ADAM(0.001)

    def run(ckpt):
        s = _solver(ude, (widths, acts), Nx, 5.0, N, 512, torch.float32, ckpt)
        out_h, st_h = s.solve_host(theta, u0)
        gu_h = np.empty((Nx, N), np.float32)
        l_h, g_h, _ = s.loss_gradient_host(theta, u0, y, grad_u0=gu_h)
        s.set_params(torch.from_numpy(theta).cuda())
        s.adam_reset()
        hist = s.train_adam(opt, torch.from_numpy(u0).cuda(), torch.from_numpy(y).cuda(), 4).cpu().numpy()
        th = s.get_params().cpu().numpy()
        out = s.forward(torch.from_numpy(u0).cuda()).cpu().numpy()
        s.close()
        return [out_h, st_h, np.float64(l_h), g_h.copy(), gu_h, hist, th, out]

    ref = run(False)
    a, b = run(True), run(True)
    assert (ref[1] == 0).all() and np.isfinite(ref[5]).all()
    for i, (r, x1, x2) in enumerate(zip(ref, a, b)):
        assert np.array_equal(x1, x2), i
        assert np.array_equal(r, x1), i


def test_script_call_checkpointing_matches_default():
    """Fisher-KPP-CNN.jl's predict_rd / loss_rd through concrete_solve with no dt (adaptive Tsit5), once with the default
    InterpolatingAdjoint and once with checkpointing = true: the two calls use different handles and give bitwise the same loss and
    gradient, in fp32 and fp64."""
    from universal_differential_equations_b200 import (FastChain, FastDense, FisherKPPUDE, InterpolatingAdjoint, ODEProblem, ReverseDiffVJP,
                                                        Tsit5, concrete_solve, initial_params, sciml)
    ude = _ude()
    X, T, dx, dt = 1.0, 5.0, 0.04, 0.5
    x = np.arange(0.0, X + dx / 2, dx)
    Nx = len(x)
    rho0 = (np.tanh((x - 0.4) / 0.02) - np.tanh((x - 0.6) / 0.02)) / 2
    data = np.random.default_rng(3).uniform(0.0, 0.5, (Nx, 11))
    rx_nn = FastChain(FastDense(1, 10, ude.tanh), FastDense(10, 20, ude.tanh), FastDense(20, 10, ude.tanh), FastDense(10, 1))
    p = np.concatenate([initial_params(rx_nn, np.random.default_rng(1)), [1.1, -2.5, 1.0], [0.0], [6.5]])
    prob_nn = ODEProblem(FisherKPPUDE(rx_nn, Nx), rho0, (0.0, T), p)
    for dtype in (torch.float32, torch.float64):
        d = torch.as_tensor(data, dtype=dtype, device="cuda")
        res = []
        for sa in (InterpolatingAdjoint(autojacvec=ReverseDiffVJP()), InterpolatingAdjoint(autojacvec=ReverseDiffVJP(), checkpointing=True)):
            before = {id(v) for v in sciml._SOLVERS.values()}
            th = torch.tensor(p, dtype=dtype, device="cuda", requires_grad=True)
            pred = concrete_solve(prob_nn, Tsit5(), rho0, th, saveat=dt, sensealg=sa, dtype=dtype)
            loss = ((d - pred) ** 2).sum() + 10 ** 2 * th[-5:-2].sum().abs()
            loss.backward()
            if sa.checkpointing:   # a handle of its own
                assert {id(v) for v in sciml._SOLVERS.values()} - before
            res.append((pred.detach().cpu().numpy(), loss.detach().cpu().numpy(), th.grad.cpu().numpy()))
        for a, b in zip(*res):
            assert np.isfinite(a).all() and np.array_equal(a, b), dtype
