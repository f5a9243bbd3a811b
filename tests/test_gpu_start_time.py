"""Every handle at a start time t0 != 0 (b200ude_desc.t0, `UDESolver(f, t0, ...)`, tspan[1] of `concrete_solve`) on the GPU.

t0 is 0 (the control), 1.7 (a shooting-window start that is no binary fraction), -1.5 (a tspan that ends at 0) and 1900 (calendar
years, where ulp(t) = 1.2e-4 in fp32).  Three kinds of check:

  - the forced model, the one model that reads t, and the adaptive Tsit5 of the runtime-shape and tensor-core LV kernels against
    the fp64 references run at the same absolute t0 (tests/test_start_time_oracle.py checks that those references honour t0), at
    the bounds of the t0 = 0 test of the same mode, cited beside each bound;
  - every other mode, adaptive and fixed step: every output (states, status, fused-L2 loss, grad theta, dL/du0) bitwise equal to
    the same handle at t0 = 0, which the existing test of that mode compares with its fp64 reference.  The autonomous models never
    read t, so their kernels run on t - t0 and t0 cannot change a bit;
  - the forced model's identity t0 = T with phases F  ==  t0 = 0 with phases F + W T (mod 2 pi), its zero initial state at
    t0 = 1900 (FENE-P's u0), and Hudson Bay through concrete_solve with tspan = (1900, 1920) in years.

Measured numbers are printed (`pytest -s`)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import forced_ref as FR  # noqa: E402
import operator_ref as OR  # noqa: E402
from helpers import glorot_theta, synthetic_ensemble  # noqa: E402
from test_start_time_oracle import shift_phases  # noqa: E402

T0S = [0.0, 1.7, -1.5, 1900.0]
F64, F32 = torch.float64, torch.float32


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _t(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def _run(s, theta, u0, y, forcing=None):
    """forward + fused L2 adjoint -> dict of numpy outputs"""
    s.set_params(_t(theta, s.dtype))
    if forcing is not None:
        s.set_forcing(_t(forcing, s.dtype))
    st = torch.full((u0.shape[1],), -1, dtype=torch.int32, device="cuda")
    out = s.forward(_t(u0, s.dtype), status=st)
    loss, g, gu = s.adjoint_l2(_t(y, s.dtype), want_grad_u0=True)
    torch.cuda.synchronize()
    return dict(out=out.cpu().double().numpy(), status=st.cpu().numpy(), loss=np.array([float(loss)]), g=g.cpu().double().numpy(),
                gu=gu.cpu().double().numpy())


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


# ================================================================ forced model against forced_ref at the same absolute t0
def _forced_case(N, seed=0):
    """the d = 3, J = 2, r = 2 case of test_forced_oracle.CASES with N ragged trajectories"""
    m = FR.Model([4, 16, 2], ["tanh", "identity"], [4, 32, 32, 3], ["tanh", "tanh", "identity"], 2)
    rng = np.random.default_rng(seed)
    theta = rng.normal(scale=0.5, size=m.P)
    u0 = rng.normal(scale=0.3, size=(m.D, N))
    coef = np.zeros((3 * m.J, N))
    for j in range(m.J):
        coef[3 * j] = rng.uniform(0.5, 2.0, N)
        coef[3 * j + 1] = rng.uniform(0.8, 2.5, N)
        coef[3 * j + 2] = rng.uniform(-1, 1, N)
    return m, theta, u0, coef


def _forced_solver(m, N, dtype, t0, adaptive, tol=(1e-6, 1e-3)):
    ude = _ude()
    f0 = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in zip(m.w0[:-1], m.w0[1:], m.a0)])
    f1 = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in zip(m.w1[:-1], m.w1[1:], m.a1)])
    f = ude.ForcedNeuralODE(dynamics=f1, readout=f0, harmonics=m.J)
    if adaptive:   # the grid of test_gpu_forced.test_fp64_adaptive_matches_reference
        return ude.UDESolver(f, t0, 0.2, 10, 1, max_trajectories=N, device="cuda:0", adaptive=True, abstol=tol[0], reltol=tol[1],
                             max_steps=4000, dtype=dtype)
    return ude.UDESolver(f, t0, 0.05, 40, 4, max_trajectories=N, device="cuda:0", dtype=dtype)   # test_fp64_fixed_step_matches_reference


def _forced_ref(m, theta, u0, coef, data, t0, adaptive, tol=(1e-6, 1e-3)):
    if not adaptive:
        out, rec = FR.forward_fixed(m, theta, u0, coef, t0, 0.05, 40, 4)
        loss, g, gu = FR.adjoint_fixed(m, theta, rec, coef, t0, 0.05, 40, 4, data, fused=True)
        return dict(out=out, loss=loss, g=g, gu=gu)
    outs, loss, g, gu = [], 0.0, np.zeros(m.P), []
    for n in range(u0.shape[1]):
        o, r, st = FR.forward_adaptive_one(m, theta, u0[:, n], coef[:, n], t0, 0.2, 11, *tol)
        assert st == 0
        ln, gn, gun = FR.adjoint_adaptive_one(m, theta, r, o, coef[:, n], t0, 0.2, 11, data[:, :, n], fused=True)
        outs.append(o)
        loss += ln
        g += gn
        gu.append(gun)
    return dict(out=np.stack(outs, axis=2), loss=loss, g=g, gu=np.stack(gu, axis=1))


def _errors(got, ref):
    return dict(out=float(np.max(np.abs(got["out"] - ref["out"]) / (1 + np.abs(ref["out"])))), loss=abs(got["loss"][0] - ref["loss"]) / abs(ref["loss"]),
                g=float(np.linalg.norm(got["g"] - ref["g"]) / np.linalg.norm(ref["g"])), gu=_rel(got["gu"], ref["gu"]))


@pytest.mark.parametrize("t0", T0S)
@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("dtype", [F64, F32])
def test_forced_vs_reference_at_t0(dtype, adaptive, t0):
    N = 37
    m, theta, u0, coef = _forced_case(N)
    data = np.random.default_rng(3).normal(size=(11, m.D + m.R, N))
    # fp32 adaptive at abstol = reltol = 1e-5, as test_gpu_parity.test_adaptive_tsit5_forward_and_adjoint_vs_oracle; fp64 adaptive at
    # 1e-8, the tolerance at which test_gpu_forced.test_fp64_adaptive_matches_reference holds the kernel to round-off
    tol = (1e-8, 1e-8) if dtype == F64 else (1e-5, 1e-5)
    if dtype == F32:   # the reference takes the coefficients the fp32 kernel is given: at t0 = 1900, w's fp32 rounding moves w t by 2e-4
        coef = coef.astype(np.float32).astype(np.float64)
    ref = _forced_ref(m, theta, u0, coef, data, t0, adaptive, tol)
    got = _run(_forced_solver(m, N, dtype, t0, adaptive, tol), theta, u0, data, forcing=coef)
    e = _errors(got, ref)
    print(f"forced {dtype} adaptive={adaptive} t0={t0}: {e}")
    assert (got["status"] == 0).all()
    if dtype == F64:   # test_gpu_forced.test_fp64_fixed_step_matches_reference / test_fp64_adaptive_matches_reference: 1e-10 / 1e-9
        b = 1e-10 if not adaptive else 1e-9
        assert max(e.values()) <= b, e
    elif not adaptive:   # test_gpu_forced.test_fp32_fixed_step_within_fp32_bounds
        assert e["out"] <= 3e-4 and e["loss"] <= 1e-4 and e["g"] <= 2e-3 and e["gu"] <= 2e-3, e
    else:                # test_gpu_parity.test_adaptive_tsit5_forward_and_adjoint_vs_oracle: 50 tol, 1e-3, 5e-3, 5e-3
        assert e["out"] <= 50 * tol[0] and e["loss"] <= 1e-3 and e["g"] <= 5e-3 and e["gu"] <= 5e-3, e


@pytest.mark.parametrize("T", [1.7, -1.5, 1900.0])
@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("dtype", [F64, F32])
def test_forced_start_time_is_a_phase_shift(dtype, adaptive, T):
    """t0 = T with phases F  ==  t0 = 0 with phases remainder(F + W T, 2 pi) computed in double: 1e-12 in fp64, and in fp32 the
    bounds of test_gpu_forced.test_fp32_fixed_step_within_fp32_bounds"""
    N = 37
    m, theta, u0, coef = _forced_case(N, seed=1)
    npd = np.float64 if dtype == F64 else np.float32
    coef = coef.astype(npd)
    data = np.random.default_rng(5).normal(size=(11, m.D + m.R, N))
    a = _run(_forced_solver(m, N, dtype, T, adaptive), theta, u0, data, forcing=coef)
    b = _run(_forced_solver(m, N, dtype, 0.0, adaptive), theta, u0, data, forcing=shift_phases(coef, m.J, T).astype(npd))
    e = {k: _rel(a[k], b[k]) for k in ("out", "loss", "g", "gu")}
    print(f"forced phase shift {dtype} adaptive={adaptive} T={T}: {e}, bitwise={all(np.array_equal(a[k], b[k]) for k in a)}")
    assert (a["status"] == 0).all() and np.array_equal(a["status"], b["status"])
    if dtype == F64:
        assert max(e.values()) <= 1e-12, e
    else:
        assert e["out"] <= 3e-4 and e["loss"] <= 1e-4 and e["g"] <= 2e-3 and e["gu"] <= 2e-3, e


def test_forced_zero_state_at_calendar_time():
    """FENE-P's u0 = 0 (NonNewtonianFluids/FENEP.jl), adaptive fp32 at t0 = 1900: the first step of the HNW heuristic is 1e-6
    there, below half an ulp of 1900 in fp32.  Status 0, finite, and the fp64 reference's values at t0 = 1900 at the bounds of
    test_gpu_parity.test_adaptive_tsit5_forward_and_adjoint_vs_oracle"""
    ude = _ude()
    m = FR.Model([2, 4, 1], ["tanh", "identity"], [2, 4, 1], ["tanh", "identity"], 1)
    rng = np.random.default_rng(2020)
    theta = rng.normal(scale=0.5, size=m.P)
    N, T, tol = 6, 1900.0, (1e-5, 1e-5)
    u0 = np.zeros((1, N))
    coef = ude.forcing_coefficients(np.full(N, 12.0), 1.0 + 0.2 * np.arange(N)).astype(np.float32).astype(np.float64)
    data = rng.normal(size=(11, 2, N))
    ref = _forced_ref(m, theta, u0, coef, data, T, True, tol)
    got = _run(_forced_solver(m, N, F32, T, True, tol), theta, u0, data, forcing=coef)
    e = _errors(got, ref)
    print(f"forced u0 = 0 at t0 = 1900, fp32 adaptive: status {got['status'].tolist()}, {e}")
    assert (got["status"] == 0).all()
    assert all(np.isfinite(got[k]).all() for k in got)
    assert e["out"] <= 50 * tol[0] and e["loss"] <= 1e-3 and e["g"] <= 5e-3 and e["gu"] <= 5e-3, e


# ================================================================ autonomous adaptive Tsit5 against the C oracle at absolute t0
@pytest.mark.parametrize("t0", T0S)
@pytest.mark.parametrize("form", ["lv5", "lv32_tc"])
def test_adaptive_tsit5_vs_oracle_at_t0(O, form, t0):
    """the oracle's ude_solve_adaptive_dense / ude_adjoint_replay on saveat = t0 + k save_dt; fp32 kernels; the bounds of
    test_gpu_parity.test_adaptive_tsit5_forward_and_adjoint_vs_oracle (lv5) and test_adaptive_tensor_core_lv32_vs_oracle_and_runtime_shape (lv32)"""
    ude = _ude()
    rng = np.random.default_rng(1)
    N, tol = 37, 1e-5
    if form == "lv5":
        chain = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in ((2, 5, "rbf"), (5, 5, "rbf"), (5, 5, "rbf"), (5, 2, "identity"))])
        m, theta = O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity")), glorot_theta((2, 5, 5, 5, 2), seed=2)
    else:
        chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
        m, theta = O.lv_model(), glorot_theta((2, 32, 32, 2), seed=1)
    u0, _ = synthetic_ensemble(N)
    y = rng.normal(size=(31, 2, N)).astype(np.float32)
    ts = t0 + 0.1 * np.arange(31)
    s = ude.UDESolver(ude.LotkaVolterraUDE(chain), t0, 0.1, 30, 1, max_trajectories=N, adaptive=True, abstol=tol, reltol=tol, max_steps=256)
    got = _run(s, theta, u0, y)
    assert (got["status"] == 0).all()
    l_ref, g_ref, gu_ref, eo = 0.0, np.zeros(len(theta)), np.zeros((2, N)), 0.0
    for k in range(N):
        o64, rec = O.solve_adaptive_dense(m, theta.astype(np.float64), u0[:, k].astype(np.float64), ts, tol, tol)
        eo = max(eo, np.abs(got["out"][:, :, k] - o64).max() / (1 + np.abs(o64).max()))
        l_ref += ((o64 - y[:, :, k]) ** 2).sum()
        gk, guk = O.adjoint_replay(m, theta.astype(np.float64), ts, rec, 2 * (o64 - y[:, :, k]))
        g_ref += gk
        gu_ref[:, k] = guk
    e = dict(out=eo, loss=abs(got["loss"][0] - l_ref) / abs(l_ref), g=float(np.linalg.norm(got["g"] - g_ref) / np.linalg.norm(g_ref)),
             gu=_rel(got["gu"], gu_ref))
    print(f"{form} adaptive fp32 t0={t0}: {e}")
    assert e["out"] <= 50 * tol + (3e-5 if form == "lv32_tc" else 0) and e["loss"] <= 1e-3 and e["g"] <= 5e-3 and e["gu"] <= 5e-3, e


# ================================================================ every other mode: bitwise the t0 = 0 handle
def _lv5_form(ude):
    return ude.LotkaVolterraUDE(ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in ((2, 5, "rbf"), (5, 5, "rbf"), (5, 5, "rbf"), (5, 2, "identity"))]))


def _lv32_form(ude):
    return ude.LotkaVolterraUDE(ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2)))


def _seir_form(ude):
    return ude.SEIRExposureUDE(ude.FastChain(ude.FastDense(3, 64, ude.tanh), ude.FastDense(64, 64, ude.tanh), ude.FastDense(64, 1)))


def _node_form(ude):
    return ude.NeuralODE(ude.FastChain(ude.FastDense(2, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 2)))


def _fkpp_form(ude, nx=26):
    return ude.FisherKPPUDE(ude.FastChain(ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)), nx)


def _operator_form(ude):
    model, theta, rng = _operator_model()
    chain = ude.FastChain(*[ude.FastDense(a, b, getattr(ude, {0: "identity", 1: "tanh"}[k])) for a, b, k in zip(model.widths[:-1], model.widths[1:], model.acts)])
    return ude.OperatorUDE(chain, model.D1, model.D2)


def _operator_model():
    """the d33_m7 shape of test_gpu_operator.SHAPES"""
    rng = np.random.default_rng(0)
    d, mw = 33, 7
    D1 = rng.normal(scale=1.0 / np.sqrt(mw), size=(d, mw))
    D2 = -np.eye(d) + rng.normal(scale=0.3 / np.sqrt(d), size=(d, d))
    model = OR.Model((d, 24, mw), (1, 0), D1, D2)
    return model, OR.glorot((d, 24, mw), rng) + 0.05 * rng.normal(size=model.P), rng


def _inputs(kind, N, P, rng):
    """(u0[d, N], y[n_save, d, N]) for a form kind"""
    if kind in ("lv", "lv32", "node"):
        u0, _ = synthetic_ensemble(N)
        return u0, rng.uniform(0.5, 4.0, (31, 2, N))
    if kind == "seir":
        u0 = np.tile(np.array([14e6 - 1e3, 0.0, 100.0, 0.0, 14e6, 0.0, 0.0])[:, None], (1, N))
        u0[2] *= rng.uniform(0.5, 1.5, N)
        return u0, rng.uniform(0, 100, (22, 7, N))
    if kind == "fkpp":
        x = np.linspace(0.0, 1.0, 26)
        half = rng.uniform(0.06, 0.2, N)
        u0 = 0.5 * (np.tanh((x[:, None] - 0.5 + half) / 0.02) - np.tanh((x[:, None] - 0.5 - half) / 0.02))
        return u0, rng.uniform(0.0, 0.5, (11, 26, N))
    u0 = rng.normal(scale=0.5, size=(33, N))
    return u0, rng.normal(scale=0.5, size=(11, 33, N))


# name: (form kind, dtypes, UDESolver keywords after (f, t0): dt, n_steps, save_every and the rest; env)
def _modes(ude):
    A = dict(adaptive=True, max_steps=1024)
    return {
        # adaptive: every kernel that reads a time
        "tsit5_adaptive_lv": ("lv", (F32, F64), (0.1, 30, 1), dict(A, abstol=1e-6, reltol=1e-6), {}),
        "tsit5_adaptive_node": ("node", (F32, F64), (0.1, 30, 1), dict(A, abstol=1e-6, reltol=1e-6), {}),
        "tsit5_adaptive_seir_runtime": ("seir", (F32, F64), (1.0, 21, 1), dict(A, abstol=1e-4, reltol=1e-4, loss_weights=(0, 1, 1, 1, 0, 0, 0)),
                                        dict(ADAPTIVE_TC="0")),
        "tsit5_adaptive_lv32_tc": ("lv32", (F32,), (0.1, 30, 1), dict(A, abstol=1e-5, reltol=1e-5), {}),
        "tsit5_adaptive_seir_tc": ("seir", (F32,), (1.0, 21, 1), dict(A, abstol=1e-4, reltol=1e-4, loss_weights=(0, 1, 1, 1, 0, 0, 0)), {}),
        "vern7_adaptive_tstops": ("lv", (F32, F64), (0.1, 30, 1), dict(A, abstol=1e-6, reltol=1e-6, alg=ude.Vern7()), {}),
        "vern7_dense_adaptive": ("lv", (F32, F64), (0.1, 30, 1), dict(A, abstol=1e-6, reltol=1e-6, alg=ude.Vern7(dense=True)), {}),
        "vern7_dense_fixed": ("lv", (F32, F64), (0.05, 60, 2), dict(alg=ude.Vern7(dense=True)), {}),
        "vern7_discrete_adaptive": ("lv", (F32, F64), (0.1, 30, 1), dict(A, abstol=1e-6, reltol=1e-6, alg=ude.Vern7(),
                                                                         sensealg=ude.ForwardDiffSensitivity()), {}),
        "vern7_dense_discrete_adaptive": ("lv", (F32, F64), (0.1, 30, 1), dict(A, abstol=1e-6, reltol=1e-6, alg=ude.Vern7(dense=True),
                                                                               sensealg=ude.ForwardDiffSensitivity()), {}),
        "fkpp_tsit5_adaptive": ("fkpp", (F32, F64), (0.5, 10, 1), dict(A), {}),
        "fkpp_vern7_discrete_adaptive": ("fkpp", (F32, F64), (0.5, 10, 1), dict(A, alg=ude.Vern7(), sensealg=ude.ForwardDiffSensitivity()), {}),
        "operator_tsit5_adaptive": ("operator", (F32, F64), (0.1, 10, 1), dict(A, abstol=1e-6, reltol=1e-3), {}),
        "operator_rkc2_adaptive": ("operator", (F32, F64), (0.1, 10, 1), dict(A, abstol=1e-6, reltol=1e-3, alg=ude.RKC2(eigen_est=60.0)), {}),
        # fixed step: kernels that never read t
        "lv32_warp_collective": ("lv32", (F32,), (0.1, 30, 1), {}, dict(FWD_WM="1", ADJ_WM="1")),
        "lv32_tensor_core": ("lv32", (F32,), (0.1, 30, 1), {}, dict(FWD_WM="0", ADJ_WM="0")),
        "lv32_auto": ("lv32", (F32,), (0.1, 30, 1), {}, {}),
        "lv5": ("lv", (F32,), (0.1, 30, 1), {}, {}),
        "seir_tc_tsit5": ("seir", (F32,), (0.5, 42, 2), dict(loss_weights=(0, 1, 1, 1, 0, 0, 0)), {}),
        "seir_tc_vern7": ("seir", (F32,), (0.5, 42, 2), dict(loss_weights=(0, 1, 1, 1, 0, 0, 0), alg=ude.Vern7()), {}),
        "fkpp16_tsit5": ("fkpp", (F32,), (0.05, 100, 10), {}, {}),
        "fkpp16_rkc2": ("fkpp", (F32,), (0.05, 100, 10), dict(alg=ude.RKC2(stages=8)), {}),
        "runtime_tsit5": ("node", (F32, F64), (0.05, 60, 2), {}, {}),
        "runtime_vern7": ("node", (F32, F64), (0.05, 60, 2), dict(alg=ude.Vern7()), {}),
        "runtime_discrete": ("node", (F32, F64), (0.05, 60, 2), dict(sensealg=ude.ForwardDiffSensitivity()), {}),
        "operator_tsit5": ("operator", (F32, F64), (0.05, 20, 2), {}, {}),
        "operator_rkc2": ("operator", (F32, F64), (0.05, 20, 2), dict(alg=ude.RKC2(stages=6)), {}),
    }


_FORMS = {"lv": _lv5_form, "lv32": _lv32_form, "seir": _seir_form, "node": _node_form, "fkpp": _fkpp_form, "operator": _operator_form}
_ADAPTIVE = ["tsit5_adaptive_lv", "tsit5_adaptive_node", "tsit5_adaptive_seir_runtime", "tsit5_adaptive_lv32_tc", "tsit5_adaptive_seir_tc",
             "vern7_adaptive_tstops", "vern7_dense_adaptive", "vern7_dense_fixed", "vern7_discrete_adaptive", "vern7_dense_discrete_adaptive",
             "fkpp_tsit5_adaptive", "fkpp_vern7_discrete_adaptive", "operator_tsit5_adaptive", "operator_rkc2_adaptive"]
_FIXED = ["lv32_warp_collective", "lv32_tensor_core", "lv32_auto", "lv5", "seir_tc_tsit5", "seir_tc_vern7", "fkpp16_tsit5", "fkpp16_rkc2",
          "runtime_tsit5", "runtime_vern7", "runtime_discrete", "operator_tsit5", "operator_rkc2"]


def _mode_outputs(name, dtype, t0, monkeypatch):
    ude = _ude()
    kind, dtypes, grid, kw, env = _modes(ude)[name]
    if dtype not in dtypes:
        pytest.skip(f"{name} has no {dtype} kernels")
    for k, v in env.items():
        monkeypatch.setenv("B200UDE_" + k, v)
    f = _FORMS[kind](ude)
    N = 37 if kind in ("seir", "fkpp", "operator") else 129
    rng = np.random.default_rng(7)
    s = ude.UDESolver(f, t0, *grid, max_trajectories=N, dtype=dtype, **kw)
    if kind == "operator":
        theta = _operator_model()[1]
    elif kind == "fkpp":
        theta = np.concatenate([glorot_theta((1, 16, 16, 1), seed=1), [1.1, -2.5, 1.0], [0.0], [6.5]])
        assert len(theta) == s.P
    else:
        theta = 0.5 * glorot_theta(f.chain.widths, seed=2) if kind == "seir" else glorot_theta(f.chain.widths, seed=2)
    u0, y = _inputs(kind, N, s.P, rng)
    y = y[:s.n_save]
    return _run(s, theta, u0, y)


@pytest.mark.parametrize("t0", [1.7, -1.5, 1900.0])
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("name", _ADAPTIVE)
def test_adaptive_autonomous_bitwise_independent_of_t0(name, dtype, t0, monkeypatch):
    base = _mode_outputs(name, dtype, 0.0, monkeypatch)
    got = _mode_outputs(name, dtype, t0, monkeypatch)
    e = {k: _rel(got[k], base[k]) if np.isfinite(got[k]).all() else float("nan") for k in ("out", "loss", "g", "gu")}
    print(f"{name} {dtype} t0={t0}: status {np.bincount(got['status'] + 1).tolist()} vs {np.bincount(base['status'] + 1).tolist()}, "
          f"rel diff {e}")
    assert (base["status"] == 0).all()
    for k in base:
        assert np.array_equal(got[k], base[k]), (k, e)


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("name", _FIXED)
def test_fixed_step_bitwise_independent_of_t0(name, dtype, monkeypatch):
    base = _mode_outputs(name, dtype, 0.0, monkeypatch)
    got = _mode_outputs(name, dtype, 1900.0, monkeypatch)
    assert (base["status"] == 0).all()
    for k in base:
        assert np.array_equal(got[k], base[k]), k


# ================================================================ the call as a user writes it
def test_hudson_bay_concrete_solve_in_calendar_years(golden):
    """hudson_bay.jl subtracts 1900 from its years; a user need not.  tspan = (1900, 1920) with saveat in years reproduces the
    reference's X-hat at the bound of test_gpu_parity.test_reference_shapes_golden_forward (3e-4 of its scale)"""
    ude = _ude()
    g = golden["hudson_bay"]
    Xhat = g["Xhat"]
    n_save = Xhat.shape[1]
    chain = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in ((2, 5, "rbf"), (5, 5, "rbf"), (5, 5, "tanh"), (5, 2, "identity"))])
    f = ude.LotkaVolterraUDE(chain, trainable_rates=2)
    years = 1900.0 + (20.0 / (n_save - 1)) * np.arange(n_save)
    prob = ude.ODEProblem(f, g["X"][:, 0].astype(np.float32), (1900.0, 1920.0), g["theta_trained"].astype(np.float32))
    for dt in (20.0 / (n_save - 1) / 8, None):   # fixed step as the golden test; adaptive (abstol = reltol = 1e-6) as a user would call it
        kw = dict(dt=dt) if dt else dict(abstol=1e-6, reltol=1e-6)
        out = ude.concrete_solve(prob, ude.Tsit5(), saveat=years, **kw).detach().cpu().double().numpy()
        e = np.abs(out - Xhat).max() / np.abs(Xhat).max()
        print(f"hudson bay in years, dt={dt}: max |X - Xhat| / max |Xhat| = {e:.3e}")
        assert out.shape == Xhat.shape and e <= 3e-4
