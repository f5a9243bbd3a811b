"""The fp64 references at a start time t0 != 0, without a GPU.  The GPU tests of tests/test_gpu_start_time.py compare every kernel
with these references at the same absolute t0, so a reference that ignored t0 (or put its save times on the wrong origin) would
certify a kernel with the same fault.  Checked here:

  - the forced model (the one non-autonomous model): the references at t0 = T equal the references at t0 = 0 with every phase
    shifted by W T (reduced mod 2 pi in double), forward and adjoint, fixed step and adaptive;
  - the autonomous models: the adaptive references at t0 = T (the C oracle's Tsit5 / Vern7 with saveat = T + k save_dt, the
    operator Tsit5 and RKC2 references, adaptive Vern7 with tstops and with dense output) equal those at t0 = 0, and their recorded
    step times start at T and are those of t0 = 0 moved by T.

T = 1900 is the worst case: there ulp(T) = 2.3e-13 in fp64, so every step length that a reference takes as a difference of two
absolute times carries a relative error of ~1e-11 for the steps here (h ~ 0.02 .. 0.1); the bounds are 1e-12 where no such
difference reaches the result, and 1e-10 where one does (stated per test)."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import discrete_ref as DR  # noqa: E402
import forced_ref as FR  # noqa: E402
import operator_ref as OR  # noqa: E402
import operator_rkc2_adaptive_ref as RA  # noqa: E402
import vern7_dense_ref as V  # noqa: E402
from helpers import glorot_theta  # noqa: E402
from test_forced_oracle import case  # noqa: E402

T0S = [1.7, -1.5, 1900.0]


def shift_phases(coef, J, T):
    """the forcing coefficients [3J, N] with phi_j -> remainder(phi_j + w_j T, 2 pi), in double (as the library folds them)"""
    c = np.array(coef, dtype=np.float64, copy=True)
    for j in range(J):
        c[3 * j + 2] = [math.remainder(float(f) + float(w) * T, 2 * math.pi) for f, w in zip(c[3 * j + 2], c[3 * j + 1])]
    return c


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


@pytest.mark.parametrize("T", T0S)
@pytest.mark.parametrize("name", ["nn", "d3_j2_r2"])
def test_forced_fixed_reference_at_t0_is_the_phase_shifted_reference(name, T):
    """gamma(T + s) = sum A cos(W s + (F + W T)): the fixed-grid forward and adjoint at t0 = T against t0 = 0 with shifted phases.
    The reference evaluates W t at absolute t, whose rounding is the only difference: ulp(W t) = 9e-13 at T = 1900 (W <= 2.5), so
    the bound is 1e-12 and 1e-14 |T| beyond that (measured 4.3e-12 at T = 1900, 5e-15 at 1.7 and -1.5)."""
    m, theta, u0, coef = case(name)
    data = np.random.default_rng(3).normal(size=(11, m.D + m.R, u0.shape[1]))
    out_t, rec_t = FR.forward_fixed(m, theta, u0, coef, T, 0.05, 40, 4)
    l_t, g_t, gu_t = FR.adjoint_fixed(m, theta, rec_t, coef, T, 0.05, 40, 4, data, fused=True)
    cs = shift_phases(coef, m.J, T)
    out_0, rec_0 = FR.forward_fixed(m, theta, u0, cs, 0.0, 0.05, 40, 4)
    l_0, g_0, gu_0 = FR.adjoint_fixed(m, theta, rec_0, cs, 0.0, 0.05, 40, 4, data, fused=True)
    e = dict(out=rel(out_t, out_0), loss=abs(l_t - l_0) / abs(l_0), g=rel(g_t, g_0), gu=rel(gu_t, gu_0))
    print(name, T, e)
    assert max(e.values()) <= max(1e-12, 1e-14 * abs(T)), e
    # and the shift is not vacuous: the unshifted forcing at t0 = 0 is another problem
    assert rel(FR.forward_fixed(m, theta, u0, coef, 0.0, 0.05, 40, 4)[0], out_0) > 1e-3


@pytest.mark.parametrize("T", T0S)
def test_forced_adaptive_reference_at_t0_is_the_phase_shifted_reference(T):
    """adaptive forward and replay adjoint, one trajectory at a time: the same number of accepted steps, the record starting at T,
    values to 1e-9.  The step times themselves agree only to ~1e-9 (T = 1.7) .. 1e-5 (T = 1900): the error estimate h sum b~_j k_j
    cancels ~8 digits at tolerance 1e-8, so the round-off of gamma at absolute t moves the PI controller's next step."""
    m, theta, u0, coef = case("d3_j2_r2")
    n_save, save_dt = 11, 0.2
    data = np.random.default_rng(4).normal(size=(n_save, m.D + m.R, u0.shape[1]))
    cs = shift_phases(coef, m.J, T)
    for n in range(u0.shape[1]):
        o_t, r_t, s_t = FR.forward_adaptive_one(m, theta, u0[:, n], coef[:, n], T, save_dt, n_save, 1e-8, 1e-8)
        o_0, r_0, s_0 = FR.forward_adaptive_one(m, theta, u0[:, n], cs[:, n], 0.0, save_dt, n_save, 1e-8, 1e-8)
        assert s_t == 0 and s_0 == 0 and r_t["nacc"] == r_0["nacc"]
        assert r_t["tgrid"][0] == T
        l_t, g_t, gu_t = FR.adjoint_adaptive_one(m, theta, r_t, o_t, coef[:, n], T, save_dt, n_save, data[:, :, n], fused=True)
        l_0, g_0, gu_0 = FR.adjoint_adaptive_one(m, theta, r_0, o_0, cs[:, n], 0.0, save_dt, n_save, data[:, :, n], fused=True)
        e = dict(out=rel(o_t, o_0), loss=abs(l_t - l_0) / abs(l_0), g=rel(g_t, g_0), gu=rel(gu_t, gu_0))
        print(T, n, r_t["nacc"], e)
        assert max(e.values()) <= 1e-9, e


def _lv5(O):
    m = O.lv_model((2, 5, 5, 5, 2), ("rbf", "rbf", "rbf", "identity"))
    return m, glorot_theta((2, 5, 5, 5, 2), seed=2).astype(np.float64), np.array([0.7, 3.1])


@pytest.mark.parametrize("T", T0S)
def test_c_oracle_adaptive_tsit5_and_replay_at_t0(O, T):
    """ude_solve_adaptive_dense / ude_adjoint_replay with saveat = T + k save_dt against saveat = k save_dt"""
    m, th, u0 = _lv5(O)
    ns, sdt = 31, 0.1
    y = np.random.default_rng(1).uniform(0.5, 4.0, (ns, 2))
    o0, r0 = O.solve_adaptive_dense(m, th, u0, sdt * np.arange(ns), 1e-6, 1e-6)
    ot, rt = O.solve_adaptive_dense(m, th, u0, T + sdt * np.arange(ns), 1e-6, 1e-6)
    assert rt[3] == r0[3] and rt[0][0] == T
    n = r0[3] + 1
    assert np.abs((rt[0][:n] - T) - r0[0][:n]).max() <= 4 * np.spacing(abs(T) + 3.0)
    g0, gu0 = O.adjoint_replay(m, th, sdt * np.arange(ns), r0, 2 * (o0 - y))
    gt, gut = O.adjoint_replay(m, th, T + sdt * np.arange(ns), rt, 2 * (ot - y))
    e = dict(out=rel(ot, o0), g=rel(gt, g0), gu=rel(gut, gu0))
    print(T, r0[3], e)
    assert max(e.values()) <= 1e-10, e
    # Vern7 stopping at every save time (the tstops path of ude_solve_adaptive)
    v0, n0, _ = O.solve_adaptive(m, th, u0, sdt * np.arange(ns), 1e-6, 1e-6, solver=O.VERN7)
    vt, nt, _ = O.solve_adaptive(m, th, u0, T + sdt * np.arange(ns), 1e-6, 1e-6, solver=O.VERN7)
    assert nt == n0 and rel(vt, v0) <= 1e-10


@pytest.mark.parametrize("T", T0S)
def test_vern7_references_at_t0(O, T):
    """adaptive Vern7 with tstops (discrete_ref) and with dense output (vern7_dense_ref), record and interpolating adjoint"""
    m, th, u0 = _lv5(O)
    ns, sdt = 31, 0.1
    dl = np.random.default_rng(2).normal(size=(ns, 2))
    a0, ra0 = DR.vern7_adaptive_record(O, m, th, u0, 0.0, sdt, ns, 1e-6, 1e-6)
    at, rat = DR.vern7_adaptive_record(O, m, th, u0, T, sdt, ns, 1e-6, 1e-6)
    assert len(rat["hstep"]) == len(ra0["hstep"]) and rat["tgrid"][0] == T
    assert np.array_equal(rat["save_step"], ra0["save_step"]) and rel(at, a0) <= 1e-10
    d0, rd0 = V.dense_record(O, m, th, u0, 0.0, sdt, ns, 1e-6, 1e-6)
    dt_, rdt = V.dense_record(O, m, th, u0, T, sdt, ns, 1e-6, 1e-6)
    assert len(rdt["hstep"]) == len(rd0["hstep"]) and rdt["tgrid"][0] == T
    g0, gu0 = V.replay_adjoint(O, m, th, rd0, 0.0, sdt, ns, dl)
    gt, gut = V.replay_adjoint(O, m, th, rdt, T, sdt, ns, dl)
    e = dict(out=rel(dt_, d0), g=rel(gt, g0), gu=rel(gut, gu0))
    print(T, len(rd0["hstep"]), e)
    assert max(e.values()) <= 1e-10, e


@pytest.mark.parametrize("T", T0S)
def test_operator_references_at_t0(T):
    """operator_ref.tsit5_adaptive(_adjoint) and operator_rkc2_adaptive_ref.rkc2_adaptive(_adjoint)"""
    rng = np.random.default_rng(0)
    d, mw = 12, 5
    D1 = rng.normal(scale=1.0 / np.sqrt(mw), size=(d, mw))
    D2 = -np.eye(d) + rng.normal(scale=0.3 / np.sqrt(d), size=(d, d))
    model = OR.Model((d, 16, mw), (1, 0), D1, D2)
    th = OR.glorot((d, 16, mw), rng)
    u0 = rng.normal(scale=0.5, size=d)
    ns, sdt = 11, 0.1
    cot = rng.normal(size=(ns, d))
    o0, r0, s0 = OR.tsit5_adaptive(model, th, u0, 0.0, sdt, ns, 1e-8, 1e-8)
    ot, rt, st = OR.tsit5_adaptive(model, th, u0, T, sdt, ns, 1e-8, 1e-8)
    assert s0 == 0 and st == 0 and len(rt[0]) == len(r0[0])
    g0, l0, _ = OR.tsit5_adaptive_adjoint(model, th, r0, 0.0, sdt, ns, o0, cot)
    gt, lt, _ = OR.tsit5_adaptive_adjoint(model, th, rt, T, sdt, ns, ot, cot)
    e = dict(out=rel(ot, o0), g=rel(gt, g0), gu=rel(lt, l0))
    print("tsit5", T, len(r0[0]), e)
    assert max(e.values()) <= 1e-10, e
    o0, r0, s0 = RA.rkc2_adaptive(model, th, u0, 0.0, sdt, ns, 1e-6, 1e-4, 40.0)
    ot, rt, st = RA.rkc2_adaptive(model, th, u0, T, sdt, ns, 1e-6, 1e-4, 40.0)
    assert s0 == 0 and st == 0 and rt[3] == r0[3] and rt[2][0] == T
    g0, l0, _ = RA.rkc2_adaptive_adjoint(model, th, r0, 0.0, sdt, ns, o0, cot)
    gt, lt, _ = RA.rkc2_adaptive_adjoint(model, th, rt, T, sdt, ns, ot, cot)
    e = dict(out=rel(ot, o0), g=rel(gt, g0), gu=rel(lt, l0))
    print("rkc2", T, len(r0[3]), e)
    assert max(e.values()) <= 1e-10, e
