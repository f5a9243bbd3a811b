"""The forced neural ODE with a readout network (B200UDE_MODEL_FORCED, NonNewtonianFluids/FENEP.jl) without a GPU:
the FENE-P truth against the reference's own record, the fp64 reference (forced_ref.py) against torch autograd through a
pure-torch Tsit5 and against finite differences, and the descriptor validation of b200ude_create."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import forced_ref as R  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fenep.npz")

# (f0 widths, f0 acts, f1 widths, f1 acts, J): the script's NN pair and linear pair (FENEP.jl:83-86), and a wider case
CASES = {
    "nn": ([2, 4, 1], ["tanh", "identity"], [2, 4, 1], ["tanh", "identity"], 1),
    "linear": ([2, 1], ["identity"], [2, 1], ["identity"], 1),
    "d3_j2_r2": ([4, 16, 2], ["tanh", "identity"], [4, 32, 32, 3], ["tanh", "tanh", "identity"], 2),
}


def case(name, seed=0):
    w0, a0, w1, a1, J = CASES[name]
    m = R.Model(w0, a0, w1, a1, J)
    rng = np.random.default_rng(seed)
    theta = rng.normal(scale=0.5, size=m.P)
    N = 3
    u0 = rng.normal(scale=0.3, size=(m.D, N))
    coef = np.zeros((3 * J, N))
    for j in range(J):
        coef[3 * j] = rng.uniform(0.5, 2.0, N)
        coef[3 * j + 1] = rng.uniform(0.8, 2.5, N)
        coef[3 * j + 2] = rng.uniform(-1, 1, N)
    return m, theta, u0, coef


def test_fenep_truth_reproduces_reference_sigma_exact():
    """plt_data.txt column 4 is sigma_exact of gamma_d = 12 cos(1.5 t) from IDA at its default reltol 1e-3: the closed-form
    reduced ODE, solved tightly, reproduces it to 2.35e-3 of max|sigma| (IDA's own error)"""
    z = np.load(GOLDEN)
    s = R.fenep_truth(z["t"], lambda t: 12 * np.cos(1.5 * t))
    err = np.abs(s - z["sigma_exact"]).max() / np.abs(z["sigma_exact"]).max()
    assert err < 3e-3, err
    # the truth is converged: halving the RK4 step changes it far below the bound
    s2 = R.fenep_truth(z["t"], lambda t: 12 * np.cos(1.5 * t), substeps=400)
    assert np.abs(s2 - s).max() < 1e-9 * np.abs(s).max()


# ---------------------------------------------------------------- torch autograd through a pure-torch Tsit5
def _torch_loss(m, theta, u0, coef, data, t0, dt, n_steps, save_every, lossw):
    def chain(th, c, x):
        h = x
        for W, b, a, off in m.layers(np.zeros(m.P), c):
            nout, nin = W.shape
            Wt = th[off:off + nin * nout].reshape(nin, nout).T
            bt = th[off + nin * nout:off + nin * nout + nout]
            z = Wt @ h + bt[:, None]
            h = torch.tanh(z) if a == "tanh" else (torch.exp(-z * z) if a == "rbf" else z)
        return h

    cf = torch.as_tensor(coef)

    def gam(t):
        g = 0.0
        for j in range(m.J):
            g = cf[3 * j] * torch.cos(cf[3 * j + 1] * t + cf[3 * j + 2]) + g
        return g

    def rows(u, t):
        return torch.cat([u, chain(theta, 0, torch.cat([u, gam(t)[None, :]]))])

    def f(u, t):
        return chain(theta, 1, torch.cat([u, gam(t)[None, :]]))

    w = torch.as_tensor(lossw)[:, None]
    u = u0
    loss = (w * (rows(u, t0) - torch.as_tensor(data[0])) ** 2).sum()
    isave = 1
    k0 = f(u, t0)
    for s in range(n_steps):
        tn = s * dt + t0
        k = [k0]
        for i in range(1, 7):
            g = u + dt * sum(float(R.TS_A[i, j]) * k[j] for j in range(i) if R.TS_A[i, j] != 0.0)
            if i == 6:
                u = g
            k.append(f(g, R.TS_C[i] * dt + tn))
        k0 = k[6]
        if (s + 1) % save_every == 0:
            loss = loss + (w * (rows(u, (s + 1) * dt + t0) - torch.as_tensor(data[isave])) ** 2).sum()
            isave += 1
    return loss


@pytest.mark.parametrize("name", list(CASES))
def test_fixed_grid_reference_matches_torch_autograd_and_finite_differences(name):
    m, theta, u0, coef = case(name)
    t0, dt, n_steps, save_every = 0.0, 0.01, 200, 20
    rng = np.random.default_rng(5)
    n_save = n_steps // save_every + 1
    data = rng.normal(size=(n_save, m.D + m.R, u0.shape[1]))
    lossw = np.linspace(0.5, 1.5, m.D + m.R)
    out, rec = R.forward_fixed(m, theta, u0, coef, t0, dt, n_steps, save_every)
    loss, g, gu0 = R.adjoint_fixed(m, theta, rec, coef, t0, dt, n_steps, save_every, data, fused=True, lossw=lossw)
    assert abs(loss - float((lossw[None, :, None] * (out - data) ** 2).sum())) <= 1e-12 * loss

    th = torch.tensor(theta, requires_grad=True)
    uu = torch.tensor(u0, requires_grad=True)
    lt = _torch_loss(m, th, uu, coef, data, t0, dt, n_steps, save_every, lossw)
    gt, gut = torch.autograd.grad(lt, (th, uu))
    assert abs(float(lt.detach()) - loss) <= 1e-10 * abs(loss)
    # interpolating adjoint (continuous) vs the exact gradient of the discrete scheme at this fine grid
    assert np.linalg.norm(g - gt.numpy()) <= 1e-5 * np.linalg.norm(gt.numpy())
    assert np.abs(gu0 - gut.numpy()).max() <= 1e-5 * np.abs(gut.numpy()).max()

    # finite differences of the reference loss along a few random directions
    for k in range(3):
        v = np.random.default_rng(10 + k).normal(size=m.P)
        v /= np.linalg.norm(v)
        e = 1e-5

        def L(tt):
            o, _ = R.forward_fixed(m, tt, u0, coef, t0, dt, n_steps, save_every)
            return float((lossw[None, :, None] * (o - data) ** 2).sum())
        fd = (L(theta + e * v) - L(theta - e * v)) / (2 * e)
        assert abs(fd - g @ v) <= 1e-5 * max(abs(fd), np.linalg.norm(g)), (fd, g @ v)


def test_adaptive_reference_replay_matches_fixed_grid_gradient():
    """the replay adjoint of an adaptive solve at tight tolerance agrees with the fixed-grid adjoint at a fine step"""
    m, theta, u0, coef = case("d3_j2_r2", seed=2)
    n_save, save_dt = 6, 0.4
    data = np.random.default_rng(1).normal(size=(n_save, m.D + m.R, u0.shape[1]))
    outf, rec = R.forward_fixed(m, theta, u0, coef, 0.0, 0.004, 500, 100)
    lf, gf, guf = R.adjoint_fixed(m, theta, rec, coef, 0.0, 0.004, 500, 100, data, fused=True)
    g = np.zeros(m.P)
    lsum = 0.0
    for n in range(u0.shape[1]):
        out, r, st = R.forward_adaptive_one(m, theta, u0[:, n], coef[:, n], 0.0, save_dt, n_save, 1e-10, 1e-10)
        assert st == 0 and np.abs(out - outf[:, :, n]).max() < 1e-7
        l, gn, gu = R.adjoint_adaptive_one(m, theta, r, out, coef[:, n], 0.0, save_dt, n_save, data[:, :, n], fused=True)
        lsum += l
        g += gn
        assert np.abs(gu - guf[:, n]).max() < 1e-6 * max(1.0, np.abs(guf).max())
    assert abs(lsum - lf) < 1e-7 * lf
    assert np.linalg.norm(g - gf) < 1e-6 * np.linalg.norm(gf)


# ---------------------------------------------------------------- descriptor validation (no device needed)
def _desc(dtype=0, w0=(2, 4, 1), a0=(1, 0), w1=(2, 4, 1), a1=(1, 0), J=1, **kw):
    from universal_differential_equations_b200 import _lib
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim = dtype, _lib.MODEL_FORCED, w1[-1]
    d.n_layers = len(a0) + len(a1)
    for i, w in enumerate(list(w0) + list(w1)):
        d.widths[i] = w
    for i, a in enumerate(list(a0) + list(a1)):
        d.acts[i] = a
    d.n_consts = 2
    d.consts[0], d.consts[1] = len(a0), J
    d.solver, d.sensealg = _lib.TSIT5, _lib.INTERPOLATING_ADJOINT
    d.t0, d.dt, d.n_steps, d.save_every = 0.0, 0.1, 10, 1
    d.max_trajectories = 8
    d.abstol, d.reltol, d.max_steps = 1e-6, 1e-3, 100
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _create(d):
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.b200ude_create(C.byref(d), C.byref(h))
    if h.value:
        L.b200ude_destroy(h)
    return rc, (L.b200ude_last_error(None) or b"").decode()


@pytest.fixture(scope="module")
def nogpu():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present (the GPU tests cover creation)")


@pytest.mark.parametrize("dtype", [0, 1])
@pytest.mark.parametrize("adaptive", [0, 1])
def test_valid_forced_descriptors_reach_the_device_check(nogpu, dtype, adaptive):
    from universal_differential_equations_b200 import _lib
    for kw in ({}, dict(w0=(4, 16, 2), w1=(4, 32, 32, 3), a1=(1, 1, 0), J=2), dict(w0=(2, 1), a0=(0,), w1=(2, 1), a1=(0,))):
        rc, msg = _create(_desc(dtype=dtype, adaptive=adaptive, **kw))
        assert rc == _lib.ENODEVICE, msg
    d = _desc(dtype=dtype, adaptive=adaptive, n_loss_weights=2)
    d.loss_weights[0], d.loss_weights[1] = 0.0, 1.0
    assert _create(d)[0] == _lib.ENODEVICE


@pytest.mark.parametrize("bad,needle", [
    (dict(w0=(3, 4, 1)), "f0's input"),
    (dict(w0=(3, 4, 1), w1=(2, 4, 2)), "f1's input"),
    (dict(w1=(2, 4, 3), state_dim=1), "f1's output"),
    (dict(J=0), "J = consts[1]"),
    (dict(J=5), "J = consts[1]"),
    (dict(w0=(2, 4, 9)), "readout width"),
    (dict(w0=(2, 65, 1)), "width"),
    (dict(n_layers=6), "L0 + L1 <= 5"),
    (dict(n_consts=1), "n_consts"),
    (dict(n_loss_weights=1), "n_loss_weights"),
    (dict(adaptive=1, abstol=0.0), "adaptive"),
])
def test_malformed_forced_descriptors_are_einval(bad, needle):
    from universal_differential_equations_b200 import _lib
    rc, msg = _create(_desc(**bad))
    assert rc == _lib.EINVAL and "MODEL_FORCED" in msg and needle in msg, msg


def test_split_that_leaves_a_chain_empty_is_einval():
    from universal_differential_equations_b200 import _lib
    d = _desc()
    d.consts[0] = 4.0   # all layers to f0
    rc, msg = _create(d)
    assert rc == _lib.EINVAL and "L0" in msg


@pytest.mark.parametrize("dtype", [0, 1])
@pytest.mark.parametrize("what", ["vern7", "rkc2", "discrete", "vern7_dense", "discrete_dense"])
def test_unbuilt_solvers_on_the_forced_model_are_unsupported(dtype, what):
    from universal_differential_equations_b200 import _lib
    kw = {"vern7": dict(solver=_lib.VERN7), "rkc2": dict(solver=_lib.RKC2, n_stages=4), "discrete": dict(sensealg=_lib.DISCRETE_ADJOINT),
          "vern7_dense": dict(solver=_lib.VERN7, flags=_lib.FLAG_VERN7_DENSE),
          "discrete_dense": dict(solver=_lib.VERN7, sensealg=_lib.DISCRETE_ADJOINT, flags=_lib.FLAG_DISCRETE_DENSE, adaptive=1)}[what]
    rc, msg = _create(_desc(dtype=dtype, **kw))
    assert rc == _lib.EUNSUPPORTED and "MODEL_FORCED" in msg, msg


def test_python_form_builds_the_back_to_back_descriptor():
    import universal_differential_equations_b200 as ude
    f0 = ude.FastChain(ude.FastDense(4, 16, ude.tanh), ude.FastDense(16, 2))
    f1 = ude.FastChain(ude.FastDense(4, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 3))
    f = ude.ForcedNeuralODE(dynamics=f1, readout=f0, harmonics=2)
    n, w, a = f.desc_layers()
    assert n == 5 and w == (4, 16, 2, 4, 32, 32, 3) and a == ("tanh", "identity", "tanh", "tanh", "identity")
    assert f.consts() == (2.0, 2.0) and f.state_dim == 3 and f.readout_dim == 2
    assert f.num_params() == R.Model([4, 16, 2], [], [4, 32, 32, 3], [], 2).P
    coef = ude.forcing_coefficients([[12.0, 12.0], [1.0, 2.0]], [[1.0, 1.2], [0.5, 0.7]])
    assert coef.shape == (6, 2) and coef[0, 1] == 12.0 and coef[1, 1] == 1.2 and coef[3, 1] == 2.0 and coef[5, 0] == 0.0
