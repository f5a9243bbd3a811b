"""GPU tests of the kernel instantiations the parity suite does not launch: non-default LV constants and loss weights on every
LV family, handles with different constant tables used in turn, odd and unpacked Fisher-KPP grids, the approx-tanh flag, and
weight regimes of the warp-collective fp16 split.  Each is compared with the fp64 CPU oracle.

Every tolerance below is either that of the existing test of the same family (tests/test_gpu_parity.py) or, for a configuration
that had none, set from an H100 run; the value measured there is written next to it.  Each test prints what it measures.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import glorot_theta, synthetic_ensemble  # noqa: E402

P_PERT = (0.7, 0.9, 0.8, 2.4)   # p1 and p4 differ from the defaults (1.3, 1.8) and from each other: a p1 <-> p4 swap shows
C_PERT = (P_PERT[0], P_PERT[3])
WEIGHTS = [(0.25, 3.0), (0.0, 1.0)]
LV32 = (2, 32, 32, 2)
LV5 = (2, 5, 5, 5, 2)
SEIR_PERTURB = (0.8, 1.3, 0.7, 1.5, 2.0, 0.6, 1.4, 0.5, 1.7)
SEIR_W = (0, 1, 1, 1, 0, 0, 0)

# tolerances of the existing tests of each family (out: |o - o64| / (1 + |o64|) elementwise; outmax: max |o - o64| / (1 + max |o64|);
# loss: relative; grad: norm-relative; gu: max-abs relative).  The comments give the largest value measured on an H100 (400 W
# power limit) with the perturbed constants and both sets of loss weights.
WM_TOL = dict(out=1e-4, loss=1e-5, grad=2e-5, gu=2e-5)       # test_lv32_warp_collective_variants_vs_oracle; out 2.4e-6, loss 1.7e-7, grad 6.5e-7, gu 9.7e-7
TC_TOL = dict(out=3e-4, loss=1e-4, grad=2e-3, gu=2e-3)       # test_lv32_forward_adjoint_vs_oracle; out 1.5e-6, loss 9.5e-8, grad 1.1e-6, gu 1.4e-6
MIX_TOL = dict(out=3e-4, loss=1e-4, grad=1e-4, gu=1e-4)      # test_lv32_families_share_the_forward_record; out 2.4e-6, grad 9.8e-7, gu 1.4e-6
LV5_TOL = dict(out=3e-4, loss=1e-4, grad=2e-3, gu=2e-3)      # test_reference_shapes_adjoint_vs_oracle; out 2.5e-7, loss 5.2e-7, grad 5.0e-7, gu 1.2e-6
F64_TOL = dict(outmax=1e-11, loss=1e-11, grad=1e-10, gu=1e-10)   # test_f64_lv_reference_shapes_vs_oracle; outmax 3.0e-16, loss 5.6e-16, grad 1.2e-15, gu 2.8e-15
DISC_TOL = dict(loss=1e-4, grad=2e-4, gu=2e-4)               # test_discrete_adjoint_forwarddiff_sensitivity_vs_oracle; loss 1.5e-7, grad 1.8e-6, gu 8.6e-7
ADAPT_TOL = dict(loss=1e-3, grad=5e-3, gu=5e-3)              # test_adaptive_tensor_core_lv32_vs_oracle_and_runtime_shape; loss 1.2e-7, grad 1.2e-6, gu 8.5e-7


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _lv32(ude, p_true=None):
    chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
    return ude.LotkaVolterraUDE(chain) if p_true is None else ude.LotkaVolterraUDE(chain, p_true=p_true)


def _lv5(ude, acts=("rbf", "rbf", "rbf"), rates=0, p_true=None):
    chain = ude.FastChain(*[ude.FastDense(a, b, c) for a, b, c in zip(LV5[:-1], LV5[1:], acts + ("identity",))])
    kw = {} if p_true is None else {"p_true": p_true}
    return ude.LotkaVolterraUDE(chain, trainable_rates=rates, **kw)


def _seir_chain(ude):
    return ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1))


def _fkpp16(ude, nx):
    return ude.FisherKPPUDE(ude.FastChain(ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)), nx)


def _env(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv("B200UDE_" + k, v)


def _run(solver, theta, u0, data, cot=None):
    """set_params, forward, fused-L2 adjoint with grad_u0 (and an explicit-cotangent adjoint) -> numpy results."""
    dt = solver.dtype
    npdt = np.float64 if dt == torch.float64 else np.float32
    solver.set_params(torch.from_numpy(np.asarray(theta, npdt)).cuda())
    status = torch.full((u0.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(np.asarray(u0, npdt)).cuda(), status=status)
    loss, g, gu = solver.adjoint_l2(torch.from_numpy(np.asarray(data, npdt)).cuda(), want_grad_u0=True)
    res = [out.cpu().numpy(), float(loss), g.cpu().numpy(), gu.cpu().numpy(), status.cpu().numpy()]
    if cot is not None:
        g2, gu2 = solver.adjoint(torch.from_numpy(np.asarray(cot, npdt)).cuda(), want_grad_u0=True)
        res += [g2.cpu().numpy(), gu2.cpu().numpy()]
    torch.cuda.synchronize()
    return res


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _errs(res, ref, out_idx=None):
    """res = (out, loss, g, gu, ...), ref = (loss, g, gu[, out]) as O.ensemble_loss_grad returns them."""
    e = dict(loss=abs(res[1] - ref[0]) / abs(ref[0]), grad=_rel(res[2], ref[1]),
             gu=float(np.abs(res[3] - ref[2]).max() / np.abs(ref[2]).max()))
    if len(ref) > 3:
        o, o64 = (res[0], ref[3]) if out_idx is None else (res[0][..., out_idx], ref[3])
        e["out"] = float((np.abs(o - o64) / (1 + np.abs(o64))).max())
        e["outmax"] = float(np.abs(o - o64).max() / (1 + np.abs(o64).max()))
    return e


def _check(tag, e, tol):
    print(f"[{tag}] " + " ".join(f"{k} {v:.2e}" for k, v in e.items()))
    for k, t in tol.items():
        assert e[k] <= t, (tag, k, e[k], t)


def _same(a, b):
    """Bitwise equality of two result lists."""
    return all((np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y) for x, y in zip(a, b))


_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


# ============================================================================================================================
# B. LV constants x loss weights x every LV kernel
# ============================================================================================================================
N_LV = 1001
LV32_FAMILIES = {
    "wm_r1g1": (dict(FWD_WM="1", ADJ_WM="1", WM_R="1", WM_G="1"), WM_TOL),
    "wm_r2g1": (dict(FWD_WM="1", ADJ_WM="1", WM_R="2", WM_G="1"), WM_TOL),
    "wm_r2g2": (dict(FWD_WM="1", ADJ_WM="1", WM_R="2", WM_G="2"), WM_TOL),
    "tc_mma_gemm": (dict(FWD_WM="0", ADJ_WM="0", ADJ_TC="2"), TC_TOL),
    "tc_ffma_gemm": (dict(FWD_WM="0", ADJ_WM="0", ADJ_TC="1"), TC_TOL),
    "packed": (dict(FWD_WM="0", ADJ_WM="0", FWD_TC="0", ADJ_TC="0"), TC_TOL),
    "packed_smem_weights": (dict(FWD_WM="0", ADJ_WM="0", FWD_TC="0", ADJ_TC="0", FWD_SMEM="1"), TC_TOL),
    "wm_fwd_tc_adj": (dict(FWD_WM="1", ADJ_WM="0"), MIX_TOL),
    "tc_fwd_wm_adj": (dict(FWD_WM="0", ADJ_WM="1"), MIX_TOL),
    "packed_fwd_wm_adj": (dict(FWD_WM="0", FWD_TC="0", ADJ_WM="1"), MIX_TOL),
}


def _lv32_inputs(N=N_LV):
    theta = glorot_theta(LV32, seed=4)
    u0, y = synthetic_ensemble(N, seed=3)
    return theta, u0, y


def _differs(res, res_default):
    """The perturbed constants reached the kernel: the results are far from those of a default-constants run."""
    assert np.abs(res[0] - res_default[0]).max() > 1e-2 * np.abs(res_default[0]).max()
    assert _rel(res[2], res_default[2]) > 1e-2


@pytest.mark.parametrize("family", list(LV32_FAMILIES))
def test_lv32_constants_and_loss_weights_vs_oracle(O, family, monkeypatch):
    env, tol = LV32_FAMILIES[family]
    _env(monkeypatch, env)
    ude = _ude()
    theta, u0, y = _lv32_inputs()
    res = []
    for w in WEIGHTS:
        s = ude.UDESolver(_lv32(ude, P_PERT), 0.0, 0.1, 30, 1, max_trajectories=N_LV, loss_weights=w)
        r = _run(s, theta, u0, y)
        s.close()
        assert (r[4] == 0).all()
        ref = _cached(("lv32", C_PERT, w), lambda: O.ensemble_loss_grad(O.lv_model(consts=C_PERT), theta.astype(np.float64), u0, y,
                                                                        np.asarray(w, np.float64), 0.1, 30, want_out=True))
        _check(f"{family} w={w}", _errs(r, ref), tol)
        res.append(r)
    assert np.array_equal(res[0][0], res[1][0])   # the forward does not read the loss weights
    s = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N_LV, loss_weights=WEIGHTS[0])
    _differs(res[0], _run(s, theta, u0, y))
    s.close()


def _lv5_inputs(rates, N=193):
    rng = np.random.default_rng(11 + rates)
    theta = 0.5 * rng.standard_normal(87 + rates)
    if rates:
        theta[:rates] = rng.uniform(0.5, 1.5, rates)
    u0, y = synthetic_ensemble(N, n_steps=20, dt=0.05, seed=5)
    return theta, u0, y


@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("rates", [0, 1])
def test_lv5_constants_and_loss_weights_vs_oracle(O, rates, dtype):
    """2-5-5-5-2 (constant-bank kernels in fp32, runtime-shape fp64 kernels): with no trainable rate both p1 and p4 come from
    the handle's constants, with one only p1 does."""
    ude = _ude()
    tdt = torch.float64 if dtype == "f64" else torch.float32
    theta, u0, y = _lv5_inputs(rates)
    if dtype == "f32":
        theta = theta.astype(np.float32)
    m = O.lv_model(LV5, ("rbf", "rbf", "rbf", "identity"), n_prefix=rates, consts=C_PERT)
    res = []
    for w in WEIGHTS:
        s = ude.UDESolver(_lv5(ude, rates=rates, p_true=P_PERT), 0.0, 0.05, 20, 1, max_trajectories=u0.shape[1], loss_weights=w, dtype=tdt)
        r = _run(s, theta, u0, y)
        s.close()
        assert (r[4] == 0).all()
        ref = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.asarray(w, np.float64), 0.05, 20, want_out=True)
        _check(f"lv5 rates={rates} {dtype} w={w}", _errs(r, ref), F64_TOL if dtype == "f64" else LV5_TOL)
        res.append(r)
    assert np.array_equal(res[0][0], res[1][0])
    s = ude.UDESolver(_lv5(ude, rates=rates), 0.0, 0.05, 20, 1, max_trajectories=u0.shape[1], loss_weights=WEIGHTS[0], dtype=tdt)
    d = _run(s, theta, u0, y)
    s.close()
    _differs(res[0], d)


@pytest.mark.parametrize("shape", ["lv32", "lv5"])
def test_lv_vern7_runtime_shape_constants_and_loss_weights(O, shape):
    """Fixed-step Vern7 on the runtime-shape kernels: the forward against the oracle's Vern7, the gradient (interpolating adjoint
    over a Tsit5 re-solve) against the oracle's Tsit5 adjoint, at the tolerances of test_vern7_fixed_step_forward_vs_oracle."""
    ude = _ude()
    N = 64
    if shape == "lv32":
        theta, (u0, y) = glorot_theta(LV32, seed=4), synthetic_ensemble(N, seed=3)
        f, fd, m = _lv32(ude, P_PERT), _lv32(ude), O.lv_model(consts=C_PERT)
    else:
        theta = _lv5_inputs(0)[0].astype(np.float32)
        u0, y = synthetic_ensemble(N, seed=3)
        f, fd, m = _lv5(ude, p_true=P_PERT), _lv5(ude), O.lv_model(LV5, ("rbf", "rbf", "rbf", "identity"), consts=C_PERT)
    res = []
    for w in WEIGHTS:
        s = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N, loss_weights=w, alg=ude.Vern7())
        r = _run(s, theta, u0, y)
        s.close()
        assert (r[4] == 0).all()
        for k in range(0, N, 9):
            ref = O.solve_fixed(m, theta.astype(np.float64), u0[:, k].astype(np.float64), 0.1, 30, solver=O.VERN7)
            assert np.abs(r[0][:, :, k] - ref).max() <= 2e-5 * (1 + np.abs(ref).max())
        ref = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.asarray(w, np.float64), 0.1, 30)
        # test_vern7_fixed_step_forward_vs_oracle; measured loss 5.4e-8, grad 2.1e-7, gu 1.2e-6
        _check(f"vern7 {shape} w={w}", _errs(r, ref), dict(loss=1e-4, grad=2e-3, gu=2e-3))
        res.append(r)
    assert np.array_equal(res[0][0], res[1][0])
    s = ude.UDESolver(fd, 0.0, 0.1, 30, 1, max_trajectories=N, loss_weights=WEIGHTS[0], alg=ude.Vern7())
    d = _run(s, theta, u0, y)
    s.close()
    _differs(res[0], d)


@pytest.mark.parametrize("shape", ["lv32", "lv5"])
def test_lv_discrete_adjoint_constants_and_loss_weights(O, shape):
    """ForwardDiffSensitivity on the tuned LV kernels against the oracle's discrete adjoint."""
    ude = _ude()
    N = 48
    if shape == "lv32":
        theta, (u0, y) = glorot_theta(LV32, seed=4), synthetic_ensemble(N, seed=3)
        f, fd, m = _lv32(ude, P_PERT), _lv32(ude), O.lv_model(consts=C_PERT)
        dt, n = 0.1, 30
    else:
        theta, u0, y = _lv5_inputs(0, N)
        theta = theta.astype(np.float32)
        f, fd, m = _lv5(ude, p_true=P_PERT), _lv5(ude), O.lv_model(LV5, ("rbf", "rbf", "rbf", "identity"), consts=C_PERT)
        dt, n = 0.05, 20
    res = []
    for w in WEIGHTS:
        s = ude.UDESolver(f, 0.0, dt, n, 1, max_trajectories=N, loss_weights=w, sensealg=ude.ForwardDiffSensitivity())
        r = _run(s, theta, u0, y)
        s.close()
        assert (r[4] == 0).all()
        ref = O.ensemble_loss_grad_discrete(m, theta.astype(np.float64), u0.astype(np.float64), y.astype(np.float64), np.asarray(w, np.float64), dt, n)
        _check(f"discrete {shape} w={w}", _errs(r, ref), DISC_TOL)
        res.append(r)
    assert np.array_equal(res[0][0], res[1][0])
    s = ude.UDESolver(fd, 0.0, dt, n, 1, max_trajectories=N, loss_weights=WEIGHTS[0], sensealg=ude.ForwardDiffSensitivity())
    d = _run(s, theta, u0, y)
    s.close()
    _differs(res[0], d)


def _adaptive_ref(O, m, theta, u0, y, ts, tol, w):
    """Oracle adaptive Tsit5 + replay adjoint of the weighted cotangent 2 w (u - y), per trajectory (small N)."""
    N = u0.shape[1]
    wv = np.asarray(w, np.float64)[None, :]
    outs, loss, g, gu = np.zeros((len(ts), u0.shape[0], N)), 0.0, 0.0, np.zeros(u0.shape)
    for k in range(N):
        o64, rec = O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol)
        r = o64 - y[:, :, k]
        loss += float((wv * r * r).sum())
        gk, guk = O.adjoint_replay(m, theta.astype(np.float64), ts, rec, 2 * wv * r)
        g = g + gk
        gu[:, k] = guk
        outs[:, :, k] = o64
    return loss, g, gu, outs


@pytest.mark.parametrize("tc", ["1", "0"])
def test_lv32_adaptive_constants_and_loss_weights(O, tc, monkeypatch):
    """Adaptive Tsit5 (tensor-core and runtime-shape kernels): the weighted cotangent is formed by launch_l2_cot."""
    monkeypatch.setenv("B200UDE_ADAPTIVE_TC", tc)
    ude = _ude()
    N, tol = 48, 1e-5
    theta, (u0, y) = glorot_theta(LV32, seed=4), synthetic_ensemble(N, seed=3)
    ts = np.linspace(0.0, 3.0, 31)
    m = O.lv_model(consts=C_PERT)
    res = []
    for w in WEIGHTS:
        s = ude.UDESolver(_lv32(ude, P_PERT), 0.0, 0.1, 30, 1, max_trajectories=N, loss_weights=w, adaptive=True, abstol=tol, reltol=tol, max_steps=256)
        r = _run(s, theta, u0, y)
        s.close()
        assert (r[4] == 0).all()
        ref = _adaptive_ref(O, m, theta, u0, y, ts, tol, w)
        assert np.all(np.abs(r[0] - ref[3]) <= 50 * tol * (1 + np.abs(ref[3]).max(axis=(0, 1))) + 3e-5)
        _check(f"adaptive tc={tc} w={w}", _errs(r, ref[:3]), ADAPT_TOL)
        res.append(r)
    assert np.array_equal(res[0][0], res[1][0])
    s = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N, loss_weights=WEIGHTS[0], adaptive=True, abstol=tol, reltol=tol, max_steps=256)
    d = _run(s, theta, u0, y)
    s.close()
    _differs(res[0], d)


# ============================================================================================================================
# C. Handles with different constant tables, used in turn on one device
# ============================================================================================================================
def _seir_inputs(N, seed, n_save):
    rng = np.random.default_rng(seed)
    u0 = np.zeros((7, N), np.float32)
    u0[0] = 0.9 * 14e6 * rng.uniform(0.9, 1.0, N)
    u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = 14e6; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    y = rng.uniform(0, 100, (n_save, 7, N)).astype(np.float32)
    return u0, y


@pytest.mark.parametrize("family", ["tc", "packed", "lv5", "seir_tc"])
def test_interleaved_handles_keep_their_constant_tables(O, family, monkeypatch):
    """Handle A has the default constants and loss weights, handle B perturbed ones.  Calls in the order A, B, A, B must each
    give what that handle gives when it runs alone: the per-translation-unit constant bank follows the handle."""
    ude = _ude()
    if family in ("tc", "packed"):
        _env(monkeypatch, dict(FWD_WM="0", ADJ_WM="0", **(dict(FWD_TC="0", ADJ_TC="0") if family == "packed" else {})))
        N = 700
        theta, u0, y = _lv32_inputs(N)

        def make(tag):
            return ude.UDESolver(_lv32(ude, P_PERT if tag == "B" else None), 0.0, 0.1, 30, 1, max_trajectories=N,
                                 loss_weights=WEIGHTS[0] if tag == "B" else None)
    elif family == "lv5":
        theta, u0, y = _lv5_inputs(0)
        theta = theta.astype(np.float32)

        def make(tag):
            return ude.UDESolver(_lv5(ude, p_true=P_PERT if tag == "B" else None), 0.0, 0.05, 20, 1, max_trajectories=u0.shape[1],
                                 loss_weights=WEIGHTS[0] if tag == "B" else None)
    else:
        N = 300
        theta = glorot_theta((3, 64, 64, 1), seed=5)
        u0, y = _seir_inputs(N, 1, 8)
        pert = tuple(a * s for a, s in zip(O.SEIR_CONSTS, SEIR_PERTURB))

        def make(tag):
            f = ude.SEIRExposureUDE(_seir_chain(ude), p_true=pert) if tag == "B" else ude.SEIRExposureUDE(_seir_chain(ude))
            return ude.UDESolver(f, 0.0, 0.25, 28, 4, max_trajectories=N, loss_weights=(0, 0.5, 2, 1, 0, 0, 0) if tag == "B" else SEIR_W)
    alone = {}
    for tag in ("A", "B"):
        s = make(tag)
        alone[tag] = _run(s, theta, u0, y)
        s.close()
    assert not np.array_equal(alone["A"][0], alone["B"][0]) and alone["A"][1] != alone["B"][1]
    handles = {"A": make("A"), "B": make("B")}
    for tag in ("A", "B", "A", "B"):
        r = _run(handles[tag], theta, u0, y)
        assert _same(r, alone[tag]), tag
    for s in handles.values():
        s.close()


# ============================================================================================================================
# D. Odd and unpacked Fisher-KPP grids on the tuned 1-16-16-1 kernels
# ============================================================================================================================
def _fkpp_inputs(nx, N, n_steps=40, every=8):
    """As test_fisher_kpp_tuned_vs_runtime_shape_kernels: asymmetric stencil taps (a left/right swap changes the result)."""
    rng = np.random.default_rng(nx)
    D0 = 0.01 * (nx - 1) ** 2
    theta = np.concatenate([glorot_theta((1, 16, 16, 1), seed=4), [1.1, -2.3, 0.9, 0.0, D0]]).astype(np.float32)
    x = np.linspace(0, 1, nx)
    u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) for d in rng.uniform(0.15, 0.5, N)],
                  axis=1).astype(np.float32)
    dt = min(2.5 / (16 * D0), 0.05)   # dt * spectral radius of the stencil <= 0.7; the reaction term bounds it on the coarse grids
    y = (np.repeat(u0[None], n_steps // every + 1, axis=0) + rng.normal(scale=0.05, size=(n_steps // every + 1, nx, N))).astype(np.float32)
    cot = rng.standard_normal(y.shape).astype(np.float32)
    return theta, u0, y, cot, dt, n_steps, every


# Nx = 3: the smallest grid, 42 trajectories per CTA (50 leave the second CTA partly filled); Nx = 25: 5 per CTA;
# Nx = 101, 129, 255: one per CTA with 27, 31 and 1 idle lanes
@pytest.mark.parametrize("nx,N", [(3, 50), (25, 7), (101, 3), (129, 3), (255, 2)])
def test_fisher_kpp_odd_grid_scalar_kernels(O, nx, N, monkeypatch):
    """Odd grids run the scalar fkpp::forward_kernel / adjoint_kernel: forward, fused-L2 loss, explicit-cotangent adjoint and
    grad_u0 against the oracle and against the runtime-shape kernels (also on the odd grid), bitwise run to run."""
    ude = _ude()
    theta, u0, y, cot, dt, n_steps, every = _fkpp_inputs(nx, N)
    m = O.fkpp_model(nx, (1, 16, 16, 1), ("tanh", "tanh", "identity"))
    res = {}
    for tuned in ("1", "0"):
        monkeypatch.setenv("B200UDE_FKPP_TUNED", tuned)
        s = ude.UDESolver(_fkpp16(ude, nx), 0.0, dt, n_steps, every, max_trajectories=N)
        r = _run(s, theta, u0, y, cot)
        assert (r[4] == 0).all()
        assert _same(_run(s, theta, u0, y, cot), r)   # fixed-order reductions
        s.close()
        res[tuned] = r
    a, b = res["1"], res["0"]
    th64 = theta.astype(np.float64)
    ref = O.ensemble_loss_grad(m, th64, u0, y, np.ones(nx), dt, n_steps, save_every=every, want_out=True)
    # test_fisher_kpp_upde_vs_oracle; measured over the five grids: out 2.5e-7, loss 9.4e-8, grad 2.8e-7, gu 6.9e-7, explicit
    # cotangent grad 5.2e-7, gu 1.4e-7
    _check(f"fkpp nx={nx} vs oracle", _errs(a, ref), dict(out=3e-4, loss=2e-4, grad=3e-3, gu=3e-3))
    assert np.all(np.abs(a[2][-5:] - ref[1][-5:]) <= 3e-3 * np.abs(ref[1][-5:]).max() + 1e-6)   # stencil taps, D0
    gc, guc = np.zeros(theta.size), np.zeros((nx, N))
    for k in range(N):
        o, dense = O.solve_fixed(m, th64, u0[:, k].astype(np.float64), dt, n_steps, save_every=every, want_dense=True)
        gk, guc[:, k] = O.adjoint_fixed(m, th64, o, dense, dt, n_steps, cot[:, :, k].astype(np.float64), save_every=every)
        gc += gk
    e = dict(grad_cot=_rel(a[5], gc), gu_cot=float(np.abs(a[6] - guc).max() / np.abs(guc).max()))
    _check(f"fkpp nx={nx} explicit cotangent vs oracle", e, dict(grad_cot=3e-3, gu_cot=3e-3))
    # test_fisher_kpp_tuned_vs_runtime_shape_kernels
    assert np.abs(a[0] - b[0]).max() <= 2e-6 * (1 + np.abs(b[0]).max())
    assert abs(a[1] - b[1]) <= 1e-5 * abs(b[1])
    for k in (2, 3, 5, 6):
        assert _rel(a[k], b[k]) <= 1e-4, k


@pytest.mark.parametrize("nx,N", [(26, 7), (256, 3)])
def test_fisher_kpp_unpacked_kernels_on_even_grids(nx, N, monkeypatch):
    """B200UDE_FKPP_PACKED=0 runs the scalar kernels on an even grid: against the packed ones."""
    ude = _ude()
    theta, u0, y, cot, dt, n_steps, every = _fkpp_inputs(nx, N)
    res = {}
    for packed in ("1", "0"):
        monkeypatch.setenv("B200UDE_FKPP_PACKED", packed)
        s = ude.UDESolver(_fkpp16(ude, nx), 0.0, dt, n_steps, every, max_trajectories=N)
        res[packed] = _run(s, theta, u0, y, cot)
        assert (res[packed][4] == 0).all()
        s.close()
    a, b = res["0"], res["1"]
    assert not _same(a, b)
    assert np.abs(a[0] - b[0]).max() <= 2e-6 * (1 + np.abs(b[0]).max())
    assert abs(a[1] - b[1]) <= 1e-5 * abs(b[1])
    for k in (2, 3, 5, 6):
        assert _rel(a[k], b[k]) <= 1e-4, k


def test_rkc2_needs_the_packed_kernels(monkeypatch):
    """RKC2 has packed kernels only: an odd grid, or B200UDE_FKPP_PACKED=0, is refused at create time."""
    ude = _ude()
    from universal_differential_equations_b200._lib import B200UDEError, EUNSUPPORTED
    with pytest.raises(B200UDEError) as e:
        ude.UDESolver(_fkpp16(ude, 25), 0.0, 0.01, 8, 2, max_trajectories=4, alg=ude.RKC2(stages=4))
    assert e.value.code == EUNSUPPORTED
    monkeypatch.setenv("B200UDE_FKPP_PACKED", "0")
    with pytest.raises(B200UDEError) as e:
        ude.UDESolver(_fkpp16(ude, 26), 0.0, 0.01, 8, 2, max_trajectories=4, alg=ude.RKC2(stages=4))
    assert e.value.code == EUNSUPPORTED


# ============================================================================================================================
# E. approx tanh (B200UDE_FLAG_APPROX_TANH)
# ============================================================================================================================
def _approx_case(ude, O, name, monkeypatch):
    """-> (make(approx) -> solver, theta, u0, y, reference (loss, g, gu, out), indices of the trajectories the reference's out has)."""
    if name.startswith("lv32"):
        env = {"lv32_wm": dict(FWD_WM="1", ADJ_WM="1"), "lv32_tc": dict(FWD_WM="0", ADJ_WM="0"),
               "lv32_packed": dict(FWD_WM="0", ADJ_WM="0", FWD_TC="0", ADJ_TC="0"), "lv32_adaptive_tc": dict(ADAPTIVE_TC="1")}[name]
        _env(monkeypatch, env)
        m = O.lv_model()
        if name == "lv32_adaptive_tc":
            N, tol = 48, 1e-5
            theta, u0, y = _lv32_inputs(N)
            ref = _adaptive_ref(O, m, theta, u0, y, np.linspace(0.0, 3.0, 31), tol, (1.0, 1.0))
            return (lambda a: ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=tol, reltol=tol,
                                            max_steps=256, approx_tanh=a)), theta, u0, y, ref, None
        theta, u0, y = _lv32_inputs()
        ref = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(2), 0.1, 30, want_out=True)
        return (lambda a: ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N_LV, approx_tanh=a)), theta, u0, y, ref, None
    if name.startswith("seir"):
        m = O.seir_model()
        theta = glorot_theta((3, 64, 64, 1), seed=2)
        w = np.asarray(SEIR_W, np.float64)
        if name == "seir_adaptive":
            N, tol = 40, 1e-4
            u0, _ = _seir_inputs(N, 17, 22)
            ts = np.linspace(0.0, 21.0, 22)
            base = np.stack([O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol)[0] for k in range(N)], axis=2)
            y = (base * (1 + 0.05 * np.random.default_rng(3).standard_normal(base.shape))).astype(np.float32)
            ref = _adaptive_ref(O, m, theta, u0, y, ts, tol, w)
            return (lambda a: ude.UDESolver(ude.SEIRExposureUDE(_seir_chain(ude)), 0.0, 1.0, 21, 1, max_trajectories=N, adaptive=True, abstol=tol,
                                            reltol=tol, max_steps=256, loss_weights=w, approx_tanh=a)), theta, u0, y, ref, None
        N = 64
        dt, n_steps, every = (0.25, 84, 4) if name == "seir_tsit5" else (0.5, 42, 2)
        u0, _ = _seir_inputs(N, 4, 22)
        th2 = theta.astype(np.float64) * 1.05   # targets: the model's own solution for a perturbed theta (residuals O(1))
        y = np.stack([O.solve_fixed(m, th2, u0[:, k].astype(np.float64), dt, n_steps, save_every=every) for k in range(N)], axis=2).astype(np.float32)
        ref = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, w, dt, n_steps, save_every=every, want_out=True)
        idx = None
        if name == "seir_vern7":   # the Vern7 forward against the oracle's Vern7; the gradient is that of the Tsit5 re-solve
            idx = np.arange(0, N, 9)
            o7 = np.stack([O.solve_fixed(m, theta.astype(np.float64), u0[:, k].astype(np.float64), dt, n_steps, solver=O.VERN7, save_every=every)
                           for k in idx], axis=2)
            ref = (ref[0], ref[1], ref[2], o7)
        alg = ude.Vern7() if name == "seir_vern7" else ude.Tsit5()
        return (lambda a: ude.UDESolver(ude.SEIRExposureUDE(_seir_chain(ude)), 0.0, dt, n_steps, every, max_trajectories=N, loss_weights=w,
                                        alg=alg, approx_tanh=a)), theta, u0, y, ref, idx
    # Fisher-KPP 1-16-16-1 on an even grid (packed kernels)
    nx = 64
    m = O.fkpp_model(nx, (1, 16, 16, 1), ("tanh", "tanh", "identity"))
    if name == "fkpp_tsit5":
        N = 5
        theta, u0, y, _, dt, n_steps, every = _fkpp_inputs(nx, N)
        ref = O.ensemble_loss_grad(m, theta.astype(np.float64), u0, y, np.ones(nx), dt, n_steps, save_every=every, want_out=True)
        return (lambda a: ude.UDESolver(_fkpp16(ude, nx), 0.0, dt, n_steps, every, max_trajectories=N, approx_tanh=a)), theta, u0, y, ref, None
    # RKC2 as test_rkc2_stabilised_solver_fisher_kpp_vs_oracle
    N, stages, dt, n_steps, every = 9, 6, 0.05, 20, 5
    D0 = 0.01 * (nx - 1) ** 2
    theta = np.concatenate([glorot_theta((1, 16, 16, 1), seed=3), [1.0, -2.0, 1.0, 0.0, D0]]).astype(np.float32)
    x = np.linspace(0, 1, nx)
    rng = np.random.default_rng(nx)
    u0 = np.stack([0.5 * (np.tanh((x - (0.5 - d / 2)) / 0.05) - np.tanh((x - (0.5 + d / 2)) / 0.05)) for d in rng.uniform(0.15, 0.5, N)], axis=1).astype(np.float32)
    y = (0.9 * np.repeat(u0[None], 5, axis=0)).astype(np.float32)
    th64 = theta.astype(np.float64)
    loss, g, gu, out = 0.0, np.zeros(theta.size), np.zeros((nx, N)), np.zeros((5, nx, N))
    for k in range(N):
        o, us, fs = O.solve_rkc2(m, th64, u0[:, k].astype(np.float64), dt, n_steps, stages, save_every=every, want_record=True)
        r = o - y[:, :, k]
        gk, gu[:, k] = O.adjoint_rkc2(m, th64, us, fs, dt, n_steps, stages, 2 * r, save_every=every)
        loss += float((r ** 2).sum()); g += gk; out[:, :, k] = o
    return (lambda a: ude.UDESolver(_fkpp16(ude, nx), 0.0, dt, n_steps, every, max_trajectories=N, alg=ude.RKC2(stages=stages),
                                    approx_tanh=a)), theta, u0, y, (loss, g, gu, out), None


# about 5x the value measured on an H100 (400 W power limit), which each comment gives as out / loss / grad
APPROX_TOL = {
    "lv32_wm": dict(out=2.5e-4, loss=6e-6, grad=3.5e-6),             # 4.9e-5 / 1.1e-6 / 6.9e-7
    "lv32_tc": dict(out=2e-4, loss=5e-6, grad=4e-6),                 # 4.0e-5 / 9.1e-7 / 7.6e-7
    "lv32_packed": dict(out=2.2e-4, loss=3.5e-6, grad=2.2e-6),       # 4.2e-5 / 7.0e-7 / 4.4e-7
    "lv32_adaptive_tc": dict(out=8.5e-5, loss=1.6e-6, grad=4.1e-6),  # 1.7e-5 / 3.1e-7 / 8.1e-7 (includes the tolerance-1e-5 solve)
    "seir_tsit5": dict(out=7.5e-6, loss=4.4e-3, grad=2.4e-3),        # 1.4e-6 / 8.8e-4 / 4.7e-4 (residuals of a 5 % theta perturbation)
    "seir_vern7": dict(out=6.5e-6, loss=6.2e-3, grad=3.4e-3),        # 1.3e-6 / 1.2e-3 / 6.7e-4
    "seir_adaptive": dict(out=2.1e-5, loss=3.6e-6, grad=4.5e-4),     # 4.1e-6 / 7.0e-7 / 8.8e-5
    "fkpp_tsit5": dict(out=5e-7, loss=2.4e-7, grad=6.6e-7),          # 1.0e-7 / 4.8e-8 / 1.3e-7 (diffusion dominates the reaction term)
    "fkpp_rkc2": dict(out=6.5e-6, loss=3.3e-7, grad=2.3e-4),         # 1.3e-6 / 6.5e-8 / 4.5e-5
}


@pytest.mark.parametrize("name", list(APPROX_TOL))
def test_approx_tanh_vs_fp64_oracle(O, name, monkeypatch):
    """approx_tanh=True runs the TM = 1 instantiation (tanh.approx.f32, 2^-11 relative error) of every family that has one.
    Against the fp64 oracle with the exact tanh; and not bitwise the exact run, so the flag reached the kernel.  A wrong
    un-fold of the warp-collective kernels' tanh argument would give an O(1) error."""
    ude = _ude()
    make, theta, u0, y, ref, idx = _approx_case(ude, O, name, monkeypatch)
    res = {}
    for a in (True, False):
        s = make(a)
        res[a] = _run(s, theta, u0, y)
        s.close()
        assert (res[a][4] == 0).all()
    r = res[True]
    o = r[0] if idx is None else r[0][:, :, idx]
    e = dict(out=float((np.abs(o - ref[3]) / (1 + np.abs(ref[3]))).max()), loss=abs(r[1] - ref[0]) / abs(ref[0]), grad=_rel(r[2], ref[1]))
    _check(f"approx tanh {name}", e, APPROX_TOL[name])
    assert not np.array_equal(r[0], res[False][0])


@pytest.mark.parametrize("name", ["lv5_tanh", "runtime_shape", "f64"])
def test_approx_tanh_is_ignored_by_the_other_kernels(name):
    """The LV 2-5-5-5-2, runtime-shape and fp64 kernels have no tanh.approx instantiation: the flag leaves their results
    bitwise unchanged (include/b200ude.h states the same next to B200UDE_FLAG_APPROX_TANH)."""
    ude = _ude()
    N = 100
    if name == "runtime_shape":
        f = ude.LotkaVolterraUDE(ude.FastChain(ude.FastDense(2, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 2)))
        theta = glorot_theta((2, 16, 16, 2), seed=2)
    else:
        f = _lv5(ude, acts=("tanh", "tanh", "tanh"))
        theta = glorot_theta(LV5, seed=2)
    u0, y = synthetic_ensemble(N, seed=1)
    dt = torch.float64 if name == "f64" else torch.float32
    res = []
    for a in (False, True):
        s = ude.UDESolver(f, 0.0, 0.1, 30, 1, max_trajectories=N, approx_tanh=a, dtype=dt)
        res.append(_run(s, theta, u0, y))
        s.close()
    assert (res[0][4] == 0).all() and _same(res[0], res[1])


# ============================================================================================================================
# F. Weight regimes of the warp-collective fp16 hi/lo split
# ============================================================================================================================
def _regime_theta(regime):
    th = glorot_theta(LV32, seed=4)
    rng = np.random.default_rng(9)
    W1, B1, W2, B2, W3, B3 = slice(0, 64), slice(64, 96), slice(96, 1120), slice(1120, 1152), slice(1152, 1216), slice(1216, 1218)
    if regime == "small":
        th *= 0.01
    elif regime == "saturated":   # both hidden layers saturate; W3 (hence the right-hand side) stays as it was
        th[W1] *= 6
        th[W2] *= 6
    elif regime == "biases":
        for sl in (B1, B2, B3):
            th[sl] = rng.uniform(-2, 2, sl.stop - sl.start)
    elif regime == "w2_500":
        # |W2| up to ~490 (2 log2(e) W2 ~ 1400, well below the fp16 limit of the scaled copy).  W1 shrinks by the same factor so
        # that the Jacobian keeps its Glorot size: with W1 kept, dt = 0.1 is far outside Tsit5's stability region.
        th[W2] *= 1600
        th[W1] /= 1600
    return th.astype(np.float32)


# measured on an H100 (400 W power limit), largest over both sets of loss weights:
#   small      out 7.0e-7, loss 1.8e-7, grad 2.5e-7, gu 1.2e-6
#   saturated  out 4.1e-6, loss 6.4e-8, grad 8.9e-7, gu 3.4e-5 -- the tensor-core family (3xTF32) measures gu 2.3e-5 against the
#              oracle as well: grad_u0 of the saturated chain carries more fp32 round-off, hence 2e-4 instead of 2e-5
#   biases     out 8.4e-7, loss 2.8e-7, grad 4.7e-7, gu 1.0e-6
#   w2_500     out 5.1e-3, loss 1.7e-4, grad 2.2e-4, gu 4.9e-4 -- the kernels' tanh has an absolute error of ~5e-7
#              (test_device_tanh_vs_fp64), which |W2| ~ 500 amplifies in the second layer; the tensor-core family measures
#              out 3.5e-3, grad 9.5e-5, gu 4.8e-4 against the oracle.  About 5x the measured values.
REGIME_TOL = {"small": WM_TOL, "saturated": dict(WM_TOL, gu=2e-4), "biases": WM_TOL,
              "w2_500": dict(out=2.5e-2, loss=1e-3, grad=1.1e-3, gu=2.5e-3)}


@pytest.mark.parametrize("w", [(1.0, 1.0), (0.0, 1.0)])
@pytest.mark.parametrize("regime", list(REGIME_TOL))
def test_warp_collective_weight_regimes(O, regime, w, monkeypatch):
    """The warp-collective kernels (fp16 hi/lo split of W2 and of the activations, power-of-two scaling of the cotangent rows
    before W2^T q2; B_t = 0 for a component with loss weight 0) outside the Glorot range, against the fp64 oracle and against
    the tensor-core family (3xTF32)."""
    ude = _ude()
    theta = _regime_theta(regime)
    _, u0, y = _lv32_inputs()
    res = {}
    for fam in ("1", "0"):
        monkeypatch.setenv("B200UDE_FWD_WM", fam)
        monkeypatch.setenv("B200UDE_ADJ_WM", fam)
        s = ude.UDESolver(_lv32(ude), 0.0, 0.1, 30, 1, max_trajectories=N_LV, loss_weights=w)
        res[fam] = _run(s, theta, u0, y)
        s.close()
        assert (res[fam][4] == 0).all()
    ref = O.ensemble_loss_grad(O.lv_model(), theta.astype(np.float64), u0, y, np.asarray(w, np.float64), 0.1, 30, want_out=True)
    e_wm, e_tc = _errs(res["1"], ref), _errs(res["0"], ref)
    print(f"[regime {regime} w={w}] tc vs oracle: " + " ".join(f"{k} {v:.2e}" for k, v in e_tc.items()))
    _check(f"regime {regime} w={w} wm vs oracle", e_wm, REGIME_TOL[regime])
    a, b = res["1"], res["0"]
    e = dict(out=float((np.abs(a[0] - b[0]) / (1 + np.abs(b[0]))).max()), grad=_rel(a[2], b[2]), gu=float(np.abs(a[3] - b[3]).max() / np.abs(b[3]).max()))
    # TC_TOL; measured up to out 3.5e-6, grad 1.0e-6, gu 9.9e-6.  For w2_500 each family carries the tanh error above: twice
    # the oracle tolerance (measured out 5.8e-3, grad 1.2e-4, gu 6.9e-4).
    tol = dict(out=5e-2, grad=2.2e-3, gu=5e-3) if regime == "w2_500" else dict(out=3e-4, grad=2e-3, gu=2e-3)
    _check(f"regime {regime} w={w} wm vs tc", e, tol)
