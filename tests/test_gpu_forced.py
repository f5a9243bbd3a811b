"""The forced neural ODE with a readout network (B200UDE_MODEL_FORCED, `ForcedNeuralODE`) on the GPU, fp64 and fp32: forward and
interpolating adjoint against the fp64 reference (tests/forced_ref.py, checked on the CPU against torch autograd and finite
differences), per-trajectory independence, the explicit cotangent, usage errors, and FENEP.jl:41-99 transcribed."""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import forced_ref as R  # noqa: E402
from test_forced_oracle import CASES, case  # noqa: E402

# measured numbers (replay gaps, training and test errors) are printed as one JSON line each (`pytest -s` shows them); with
# B200UDE_TEST_RECORD_DIR set they are also written there as JSON files.  The tests never write into the source tree.
RECORD_DIR = os.environ.get("B200UDE_TEST_RECORD_DIR")


def _record(name, obj):
    print(json.dumps({name: obj}))
    if RECORD_DIR:
        os.makedirs(RECORD_DIR, exist_ok=True)
        with open(os.path.join(RECORD_DIR, name + ".json"), "w") as fh:
            json.dump(obj, fh)


def _ude():
    import universal_differential_equations_b200 as ude
    return ude


def _form(m):
    ude = _ude()
    w0, a0, w1, a1, J = m.w0, m.a0, m.w1, m.a1, m.J
    f0 = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in zip(w0[:-1], w0[1:], a0)])
    f1 = ude.FastChain(*[ude.FastDense(a, b, s) for a, b, s in zip(w1[:-1], w1[1:], a1)])
    return ude.ForcedNeuralODE(dynamics=f1, readout=f0, harmonics=J)


def _solver(m, N, dtype, adaptive=False, t0=0.0, dt=0.05, n_steps=40, save_every=4, abstol=1e-6, reltol=1e-3, lossw=None, max_steps=4000):
    return _ude().UDESolver(_form(m), t0, dt, n_steps, save_every, max_trajectories=N, device="cuda:0", adaptive=adaptive, abstol=abstol,
                            reltol=reltol, max_steps=max_steps, loss_weights=lossw, dtype=dtype)


def _t(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).cuda()


def _run(s, theta, u0, coef, data, dtype, cot=None):
    s.set_params(_t(theta, dtype))
    s.set_forcing(_t(coef, dtype))
    out = s.forward(_t(u0, dtype))
    loss, g, gu0 = s.adjoint_l2(_t(data, dtype), want_grad_u0=True)
    torch.cuda.synchronize()
    return out.cpu().double().numpy(), float(loss), g.cpu().double().numpy(), gu0.cpu().double().numpy()


def _ref_adaptive(m, theta, u0, coef, data, save_dt, n_save, abstol, reltol, lossw=None):
    outs, loss, g, gu = [], 0.0, np.zeros(m.P), []
    for n in range(u0.shape[1]):
        o, r, st = R.forward_adaptive_one(m, theta, u0[:, n], coef[:, n], 0.0, save_dt, n_save, abstol, reltol)
        assert st == 0
        l, gn, gun = R.adjoint_adaptive_one(m, theta, r, o, coef[:, n], 0.0, save_dt, n_save, data[:, :, n], fused=True, lossw=lossw)
        outs.append(o)
        loss += l
        g += gn
        gu.append(gun)
    return np.stack(outs, axis=2), loss, g, np.stack(gu, axis=1)


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("name", list(CASES))
def test_fp64_fixed_step_matches_reference(name):
    m, theta, u0, coef = case(name)
    N = u0.shape[1]
    data = np.random.default_rng(3).normal(size=(11, m.D + m.R, N))
    lossw = np.linspace(0.5, 1.5, m.D + m.R)
    out_r, rec = R.forward_fixed(m, theta, u0, coef, 0.0, 0.05, 40, 4)
    l_r, g_r, gu_r = R.adjoint_fixed(m, theta, rec, coef, 0.0, 0.05, 40, 4, data, fused=True, lossw=lossw)
    s = _solver(m, N, torch.float64, lossw=lossw)
    out, l, g, gu = _run(s, theta, u0, coef, data, torch.float64)
    assert np.abs(out - out_r).max() <= 1e-10 * max(1.0, np.abs(out_r).max())
    assert abs(l - l_r) <= 1e-10 * abs(l_r)
    assert _rel(g, g_r) <= 1e-10 and np.abs(gu - gu_r).max() <= 1e-10 * np.abs(gu_r).max()


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("tol", [(1e-6, 1e-3), (1e-8, 1e-8)])
def test_fp64_adaptive_matches_reference(name, tol):
    """outputs agreeing to round-off (not to the tolerance) mean the same accepted steps"""
    m, theta, u0, coef = case(name)
    N, n_save, save_dt = u0.shape[1], 11, 0.2
    data = np.random.default_rng(4).normal(size=(n_save, m.D + m.R, N))
    out_r, l_r, g_r, gu_r = _ref_adaptive(m, theta, u0, coef, data, save_dt, n_save, *tol)
    s = _solver(m, N, torch.float64, adaptive=True, dt=save_dt, n_steps=n_save - 1, save_every=1, abstol=tol[0], reltol=tol[1])
    out, l, g, gu = _run(s, theta, u0, coef, data, torch.float64)
    # measured on an H100: one trajectory of the d = 3 case at (1e-6, 1e-3) leaves round-off agreement (3.6e-7 of the state
    # scale, still 3 decades inside the tolerance): its accepted-step sequence differs from the reference's somewhere
    b, bg = (1e-6, 1e-4) if (name == "d3_j2_r2" and tol == (1e-6, 1e-3)) else (1e-9, 1e-9)
    assert np.abs(out - out_r).max() <= b * max(1.0, np.abs(out_r).max())
    assert abs(l - l_r) <= b * abs(l_r)
    assert _rel(g, g_r) <= bg and np.abs(gu - gu_r).max() <= bg * np.abs(gu_r).max()


@pytest.mark.parametrize("name", list(CASES))
def test_fp32_fixed_step_within_fp32_bounds(name):
    m, theta, u0, coef = case(name)
    N = u0.shape[1]
    data = np.random.default_rng(3).normal(size=(11, m.D + m.R, N))
    out_r, rec = R.forward_fixed(m, theta, u0, coef, 0.0, 0.05, 40, 4)
    l_r, g_r, gu_r = R.adjoint_fixed(m, theta, rec, coef, 0.0, 0.05, 40, 4, data, fused=True)
    s = _solver(m, N, torch.float32)
    out, l, g, gu = _run(s, theta.astype(np.float32), u0, coef, data, torch.float32)
    assert np.all(np.abs(out - out_r) <= 3e-4 * (1 + np.abs(out_r)))
    assert abs(l - l_r) <= 1e-4 * abs(l_r)
    assert _rel(g, g_r) <= 2e-3 and np.abs(gu - gu_r).max() <= 2e-3 * np.abs(gu_r).max()


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_trajectories_are_independent_bitwise(dtype):
    """N = 40 with per-trajectory forcing (mixed step counts): each trajectory's outputs, status and grad_u0 are bitwise those
    of the trajectory solved alone; a permutation permutes them bitwise; two runs are bitwise equal"""
    m, theta, _, _ = case("nn")
    N, n_save, save_dt = 40, 21, 0.3
    rng = np.random.default_rng(7)
    u0 = rng.normal(scale=0.3, size=(1, N))
    coef = np.stack([rng.uniform(1, 12, N), rng.uniform(0.2, 4.0, N), rng.uniform(-1, 1, N)])
    data = rng.normal(size=(n_save, 2, N))
    s = _solver(m, N, dtype, adaptive=True, dt=save_dt, n_steps=n_save - 1, save_every=1)

    def go(idx):
        s.set_params(_t(theta, dtype))
        s.set_forcing(_t(coef[:, idx], dtype))
        st = torch.zeros(len(idx), dtype=torch.int32, device="cuda")
        out = s.forward(_t(u0[:, idx], dtype), status=st)
        _, _, gu = s.adjoint_l2(_t(data[:, :, idx], dtype), want_grad_u0=True)
        torch.cuda.synchronize()
        return out.cpu().numpy(), st.cpu().numpy(), gu.cpu().numpy()

    full = go(np.arange(N))
    again = go(np.arange(N))
    for a, b in zip(full, again):
        assert np.array_equal(a, b)
    perm = rng.permutation(N)
    p = go(perm)
    assert np.array_equal(p[0], full[0][:, :, perm]) and np.array_equal(p[1], full[1][perm]) and np.array_equal(p[2], full[2][:, perm])
    for n in (0, 13, 39):
        one = go(np.array([n]))
        assert np.array_equal(one[0][:, :, 0], full[0][:, :, n]) and one[1][0] == full[1][n] and np.array_equal(one[2][:, 0], full[2][:, n])


@pytest.mark.parametrize("adaptive", [False, True])
def test_explicit_cotangent_is_linear_and_matches_fused_l2(adaptive):
    m, theta, u0, coef = case("d3_j2_r2")
    N = u0.shape[1]
    dt = torch.float64
    s = _solver(m, N, dt, adaptive=adaptive, dt=0.2 if adaptive else 0.05, n_steps=10 if adaptive else 40, save_every=1 if adaptive else 4)
    s.set_params(_t(theta, dt))
    s.set_forcing(_t(coef, dt))
    out = s.forward(_t(u0, dt))
    rng = np.random.default_rng(9)
    c1 = _t(rng.normal(size=out.shape), dt)
    c1[:, :m.D] = 0          # readout rows only
    c2 = _t(rng.normal(size=out.shape), dt)
    c2[:, m.D:] = 0          # state rows only
    g1, u1 = s.adjoint(c1)
    g2, u2 = s.adjoint(c2)
    g12, u12 = s.adjoint(c1 + 2 * c2)
    assert torch.allclose(g12, g1 + 2 * g2, rtol=1e-12, atol=1e-12 * float(g12.abs().max()))
    assert torch.allclose(u12, u1 + 2 * u2, rtol=1e-12, atol=1e-12 * float(u12.abs().max()))
    assert float(g1.abs().max()) > 0 and float(u1.abs().max()) > 0
    data = _t(rng.normal(size=out.shape), dt)
    loss, gl, gul = s.adjoint_l2(data, want_grad_u0=True)
    ge, gue = s.adjoint(2 * (out - data))
    assert abs(float(loss) - float(((out - data) ** 2).sum())) <= 1e-12 * float(loss)
    assert torch.allclose(gl, ge, rtol=1e-12, atol=1e-12 * float(ge.abs().max()))
    assert torch.allclose(gul, gue, rtol=1e-12, atol=1e-12 * float(gue.abs().max()))


def test_usage_errors():
    ude = _ude()
    from universal_differential_equations_b200 import _lib
    m, theta, u0, coef = case("nn")
    s = _solver(m, 8, torch.float32)
    s.set_params(_t(theta, torch.float32))
    with pytest.raises(_lib.B200UDEError) as e:
        s.forward(_t(u0, torch.float32))
    assert e.value.code == _lib.ESTATE
    s.set_forcing(_t(coef[:, :2], torch.float32))
    with pytest.raises(_lib.B200UDEError) as e:
        s.forward(_t(u0, torch.float32))   # 3 trajectories, forcing for 2
    assert e.value.code == _lib.ESTATE
    s.set_forcing(coef)                    # host memory
    assert s.forward(_t(u0, torch.float32)).shape == (11, 2, 3)
    chain = ude.FastChain(ude.FastDense(2, 8, ude.tanh), ude.FastDense(8, 2))
    lv = ude.UDESolver(ude.LotkaVolterraUDE(chain), 0.0, 0.1, 10, 1, max_trajectories=4, device="cuda:0")
    with pytest.raises(_lib.B200UDEError) as e:
        lv.set_forcing(coef)
    assert e.value.code == _lib.EUNSUPPORTED


# ---------------------------------------------------------------- FENEP.jl:41-99 transcribed
T1 = float(np.float32(6.2831))
OMEGAS = [float(np.float32(1.0) + i * np.float32(0.2)) for i in range(6)]   # 1.0f0:0.2f0:2.0f0


def _fenep_setup(kind, dtype):
    ude = _ude()
    if kind == "nn":
        f0 = ude.FastChain(ude.FastDense(2, 4, ude.tanh), ude.FastDense(4, 1))
        f1 = ude.FastChain(ude.FastDense(2, 4, ude.tanh), ude.FastDense(4, 1))
    else:
        f0 = ude.FastChain(ude.FastDense(2, 1))
        f1 = ude.FastChain(ude.FastDense(2, 1))
    f = ude.ForcedNeuralODE(dynamics=f1, readout=f0)
    rng = np.random.default_rng(2020)
    theta = np.concatenate([ude.initial_params(f0, rng), ude.initial_params(f1, rng)]).astype(np.float64)
    tsave = np.linspace(0.0, T1, 100)
    sig = np.stack([R.fenep_truth(tsave, lambda t, w=w: 12.0 * np.cos(w * t)) for w in OMEGAS], axis=1)   # [100, 6]
    data = np.zeros((100, 2, 6))
    data[:, 1] = sig
    coef = ude.forcing_coefficients(np.full(6, 12.0), np.array(OMEGAS))
    s = ude.UDESolver(f, 0.0, T1 / 99, 99, 1, max_trajectories=6, device="cuda:0", adaptive=True, abstol=1e-6, reltol=1e-3,
                      loss_weights=(0.0, 1.0), max_steps=4000, dtype=dtype)
    m = R.Model(list(f0.widths), list(f0.acts), list(f1.widths), list(f1.acts), 1)
    return s, m, theta, data, coef


def _adam(th, g, mm, vv, it, eta=0.015, b1=0.9, b2=0.999, eps=1e-8):
    mm[:] = b1 * mm + (1 - b1) * g
    vv[:] = b2 * vv + (1 - b2) * g * g
    return th - eta * (mm / (1 - b1 ** it)) / (np.sqrt(vv / (1 - b2 ** it)) + eps)


@pytest.mark.parametrize("kind", ["nn", "linear"])
def test_fenep_first_iterations_match_cpu_replay(kind):
    """ADAM(0.015) from a seeded Glorot init: the first 20 losses of the GPU loop equal the CPU reference's replay of the same
    iterations.  Bounds measured on an H100: the linear pair agrees to 8e-9 in fp64 and 2.2e-4 in fp32, the NN pair to 1.5e-4 in fp32.  For the NN pair the fp64
    loss already differs by 3e-8 at iteration 1 (same theta), so the adaptive step sequence differs from the reference's
    somewhere; that difference grows to 6e-5 over 20 ADAM iterations"""
    iters = 20
    _, m, theta0, data, coef = _fenep_setup(kind, torch.float64)
    u0 = np.zeros((1, 6))
    # CPU replay
    th, mm, vv, ref = theta0.copy(), np.zeros(m.P), np.zeros(m.P), []
    for it in range(1, iters + 1):
        _, l, g, _ = _ref_adaptive(m, th, u0, coef, data, T1 / 99, 100, 1e-6, 1e-3, lossw=np.array([0.0, 1.0]))
        ref.append(l)
        th = _adam(th, g, mm, vv, it)
    res = {}
    bounds = {"linear": (1e-8, 1e-3), "nn": (2e-4, 1e-3)}[kind]   # fp32 measured: 2.2e-4 (linear), 1.5e-4 (NN)
    for dtype, bound in zip((torch.float64, torch.float32), bounds):
        s = _fenep_setup(kind, dtype)[0]
        th, mm, vv, got = theta0.copy(), np.zeros(m.P), np.zeros(m.P), []
        s.set_forcing(_t(coef, dtype))
        for it in range(1, iters + 1):
            s.set_params(_t(th, dtype))
            s.forward(_t(u0, dtype))
            loss, g, _ = s.adjoint_l2(_t(data, dtype))
            got.append(float(loss))
            th = _adam(th, g.cpu().double().numpy(), mm, vv, it)
        rel = np.abs(np.array(got) - ref) / np.abs(ref)
        res[str(dtype)] = float(rel.max())
        assert rel.max() <= bound, (dtype, rel)
    _record(f"fenep_replay_{kind}", {"ref_losses": ref, "max_rel": res})


def test_fenep_training_orders_as_the_reference_record():
    """5000 ADAM(0.015) iterations of both model pairs on the device (fp32, b200ude_train_adam).  The reference's init is random
    and unrecorded, so its numbers (er_data.txt) are a comparison only; asserted is the ordering that record shows: the NN's
    training error is below the linear model's by iteration 500, and its test error (gamma_d = 12 cos(1.5 t) on (0, 10)) at 5000"""
    ude = _ude()
    tt = np.linspace(0.0, 10.0, 100)
    sig_test = R.fenep_truth(tt, lambda t: 12.0 * np.cos(1.5 * t))
    rec = {}
    for kind in ("nn", "linear"):
        s, m, theta0, data, coef = _fenep_setup(kind, torch.float32)
        s.set_forcing(_t(coef, torch.float32))
        s.set_params(_t(theta0, torch.float32))
        s.adam_reset()
        hist = s.train_adam(ude.ADAM(0.015), _t(np.zeros((1, 6)), torch.float32), _t(data, torch.float32), 5000).cpu().double().numpy()
        th = s.get_params()
        tsol = _ude().UDESolver(s.f, 0.0, 10.0 / 99, 99, 1, max_trajectories=1, device="cuda:0", adaptive=True, abstol=1e-6, reltol=1e-3,
                                max_steps=4000)
        tsol.set_params(th)
        tsol.set_forcing(ude.forcing_coefficients([12.0], [1.5]))
        out = tsol.forward(_t(np.zeros((1, 1)), torch.float32)).cpu().double().numpy()
        test_err = float(((out[:, 1, 0] - sig_test) ** 2).sum())
        rec[kind] = {"train_500": float(hist[500]), "train_5000": float(hist[-1]), "test_5000": test_err}
    _record("fenep_training", rec)
    assert np.isfinite([v for r in rec.values() for v in r.values()]).all()
    assert rec["nn"]["train_500"] < rec["linear"]["train_500"]
    assert rec["nn"]["test_5000"] < rec["linear"]["test_5000"]
