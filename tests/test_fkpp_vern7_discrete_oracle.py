"""Adaptive Vern7 with the discrete adjoint (ForwardDiffSensitivity) on the Fisher-KPP UPDE -- scenario_3.jl:121-126 as written.
The fp64 reference the GPU kernels are compared against is tests/discrete_ref.py (vern7_adaptive_record, adjoint_steps) on the
oracle's Fisher-KPP right-hand side.  Here it is checked against torch autograd through the frozen Vern7 steps, and the
script's ADAM(0.1) phase is replayed against the stored loss history (KAT-11 with the script's own sensitivity); and the
descriptor validation of the new configuration without a GPU."""
import ctypes as C

import numpy as np
import pytest

import discrete_ref as R
from helpers import glorot_theta

RBF3 = ("rbf", "rbf", "rbf", "identity")
TANH3 = ("tanh", "tanh", "tanh", "identity")


def _torch_fkpp_rhs(widths, acts):
    """The oracle's Fisher-KPP right-hand side in torch: the chain on every point, D0 * (w1 u_{i-1} + w2 u_i + w3 u_{i+1})."""
    import torch

    def f(th, u):
        x, o = u[None, :], 0
        for nin, nout, act in zip(widths[:-1], widths[1:], acts):
            W = th[o:o + nin * nout].reshape(nin, nout).T
            b = th[o + nin * nout:o + nin * nout + nout]
            o += nin * nout + nout
            a = W @ x + b[:, None]
            x = torch.tanh(a) if act == "tanh" else (torch.exp(-a * a) if act == "rbf" else a)
        P = th.shape[0]
        w1, w2, w3, D0 = th[P - 5], th[P - 4], th[P - 3], th[P - 1]
        return x[0] + D0 * (w1 * torch.roll(u, 1) + w2 * u + w3 * torch.roll(u, -1))
    return f


def _torch_loss(O, rhs, th, u0, rec, y):
    """L = sum_i |u(t_i) - y_i|^2 through Vern7 on the frozen steps rec['hstep'] (torch fp64)."""
    A, b, S, _ = R.tableau(O, R.VERN7)
    at = {int(s): i for i, s in enumerate(rec["save_step"])}
    u = u0
    L = ((u - y[0]) ** 2).sum()
    for n, h in enumerate(rec["hstep"]):
        ks = []
        for i in range(S):
            g = u + float(h) * sum(float(A[i, j]) * ks[j] for j in range(i) if A[i, j] != 0) if i else u
            ks.append(rhs(th, g))
        u = u + float(h) * sum(float(b[j]) * ks[j] for j in range(S) if b[j] != 0)
        if n in at:
            L = L + ((u - y[at[n]]) ** 2).sum()
    return L


def _pulses(Nx, widths):
    """scenario_3.jl's rho_ic(Delta) for a few widths Delta: u0[Nx] per width."""
    x = np.linspace(0.0, 1.0, Nx)
    return [(np.tanh((x - (0.5 - d / 2)) / (d / 10)) - np.tanh((x - (0.5 + d / 2)) / (d / 10))) / 2 for d in widths]


MODELS = [  # Nx, widths, acts, T
    (26, (1, 5, 5, 5, 1), RBF3, 5.0),          # the script's grid and chain
    (40, (1, 10, 20, 10, 1), TANH3, 2.0),
]


@pytest.mark.parametrize("model", MODELS, ids=["rbf26", "tanh40"])
def test_fkpp_discrete_adjoint_matches_autograd_through_the_scheme(O, model):
    torch = pytest.importorskip("torch")
    Nx, widths, acts, T = model
    m = O.fkpp_model(Nx, widths, acts)
    theta = np.concatenate([glorot_theta(widths, seed=3).astype(np.float64), [0.9, -2.1, 1.2, 0.3, 0.01 * (Nx - 1) ** 2]])
    assert len(theta) == O.num_params(m)
    u0 = _pulses(Nx, [0.4])[0]
    rhs = _torch_fkpp_rhs(widths, acts)
    g_ = u0 + 0.1 * np.sin(np.arange(Nx))
    assert np.allclose(rhs(torch.tensor(theta), torch.tensor(g_)).numpy(), O.rhs(m, theta, g_), rtol=1e-13, atol=1e-13)
    out, rec = R.vern7_adaptive_record(O, m, theta, u0, 0.0, T / 10, 11, 1e-6, 1e-3)
    assert len(rec["hstep"]) > 10   # the controller took steps between the save points
    y = np.random.default_rng(1).uniform(0.0, 0.5, out.shape)
    outs, ustep = R.solve_steps(O, m, theta, u0, rec, R.VERN7)
    assert np.abs(outs - out).max() <= 1e-12 * np.abs(out).max()
    g, gu = R.adjoint_steps(O, m, theta, ustep, rec, R.VERN7, 2 * (out - y))
    th = torch.tensor(theta, requires_grad=True)
    U0 = torch.tensor(u0, requires_grad=True)
    L = _torch_loss(O, rhs, th, U0, rec, torch.tensor(y))
    L.backward()
    # the oracle (C) and torch evaluate the chain with different libm calls: the two losses agree to round-off, not bitwise
    assert abs(float(L.detach()) - float(((out - y) ** 2).sum())) <= 1e-10 * float(L.detach())
    gt, gut = th.grad.numpy(), U0.grad.numpy()
    # torch and the oracle evaluate tanh / exp with different libm code, so the two forwards differ in the last bits and the
    # gradients by what the scheme amplifies that to: 2.1e-12 (rbf26) and 3.8e-11 (tanh40) in grad_theta, 4.7e-11 and 5.4e-11 in
    # grad_u0.  The D0 entry is a sum of cancelling terms (1.6 against entries of 3e4): it is checked on the gradient's scale.
    assert np.linalg.norm(g - gt) <= 1e-10 * np.linalg.norm(gt)
    for j in (-5, -4, -3, -1):   # w1, w2, w3, D0 on their own
        assert abs(g[j] - gt[j]) <= 1e-10 * np.linalg.norm(gt), j   # measured: at most 2.4e-11
    assert g[-2] == 0.0   # the conv bias does not enter the right-hand side
    assert np.linalg.norm(gu - gut) <= 1e-10 * np.linalg.norm(gut)


def test_kat11_adam_replay_with_the_scripts_own_sensitivity(O, golden):
    """scenario_3.jl:121-143 as written: Vern7 at the default tolerances (1e-6 / 1e-3), saveat = 0.5, ForwardDiffSensitivity,
    loss sum(abs2, pred - Xn) + |w1 + w2 + w3|, ADAM(0.1) from the stored initial parameters.  The discrete gradient of that
    solve reproduces the stored losses[0..9] (measured: at most 2.5e-6 relative)."""
    g = golden["scenario_3"]
    m = O.fkpp_model(26, (1, 5, 5, 5, 1), RBF3)
    th = g["theta_init"].astype(np.float64)
    X = g["X"].T.astype(np.float64)
    mm, vv = np.zeros_like(th), np.zeros_like(th)
    b1, b2, eta, eps = 0.9, 0.999, 0.1, 1e-8
    for it in range(1, 11):
        out, rec = R.vern7_adaptive_record(O, m, th, X[0], 0.0, 0.5, 11, 1e-6, 1e-3)
        taps = th[-5:-2].sum()
        l = ((out - X) ** 2).sum() + abs(taps)
        assert abs(l - g["losses"][it - 1]) <= 1e-5 * g["losses"][it - 1], (it, l, g["losses"][it - 1])
        gr, _ = R.adjoint_steps(O, m, th, rec["ustep"], rec, R.VERN7, 2 * (out - X))
        gr[-5:-2] += np.sign(taps)
        mm = b1 * mm + (1 - b1) * gr
        vv = b2 * vv + (1 - b2) * gr * gr
        th = th - eta * (mm / (1 - b1**it)) / (np.sqrt(vv / (1 - b2**it)) + eps)


def _desc(_lib, dtype, solver, adaptive, sensealg, Nx=26, widths=(1, 5, 5, 5, 1), acts=(2, 2, 2, 0)):
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim, d.n_layers, d.n_suffix = dtype, _lib.MODEL_FKPP, Nx, len(widths) - 1, 5
    for i, w in enumerate(widths):
        d.widths[i] = w
    for i, a in enumerate(acts):
        d.acts[i] = a
    d.solver, d.adaptive, d.sensealg = solver, adaptive, sensealg
    d.dt, d.n_steps, d.save_every, d.max_trajectories = 0.5, 10, 1, 8
    d.abstol, d.reltol, d.max_steps = 1e-6, 1e-3, 512
    if solver == _lib.RKC2:
        d.n_stages = 8
    return d


def test_fkpp_vern7_discrete_descriptors_without_a_gpu():
    """Adaptive Vern7 + discrete adjoint on Fisher-KPP passes validation in fp32 and fp64 (ENODEVICE here), the tuned 1-16-16-1
    chain on 256 points included; the other Fisher-KPP solver / sensitivity pairs stay EUNSUPPORTED."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    D, I = _lib.DISCRETE_ADJOINT, _lib.INTERPOLATING_ADJOINT
    for dtype in (_lib.F32, _lib.F64):
        for kw in ({}, dict(Nx=256, widths=(1, 16, 16, 1), acts=(1, 1, 0)), dict(Nx=3, widths=(1, 64, 64, 1), acts=(1, 1, 0))):
            rc = L.b200ude_create(C.byref(_desc(_lib, dtype, _lib.VERN7, 1, D, **kw)), C.byref(h))
            assert rc == _lib.ENODEVICE and not h.value, (dtype, kw, L.b200ude_last_error(None))
        for solver, adaptive in ((_lib.TSIT5, 0), (_lib.VERN7, 0), (_lib.TSIT5, 1), (_lib.RKC2, 0)):
            rc = L.b200ude_create(C.byref(_desc(_lib, dtype, solver, adaptive, D)), C.byref(h))
            assert rc == _lib.EUNSUPPORTED, (dtype, solver, adaptive)
            msg = L.b200ude_last_error(None)
            assert b"fixed-step Tsit5" in msg and b"adaptive Vern7" in msg, msg
        for adaptive in (0, 1):   # Vern7 with the interpolating adjoint
            assert L.b200ude_create(C.byref(_desc(_lib, dtype, _lib.VERN7, adaptive, I)), C.byref(h)) == _lib.EUNSUPPORTED, (dtype, adaptive)
    assert L.b200ude_create(C.byref(_desc(_lib, _lib.F64, _lib.TSIT5, 0, I)), C.byref(h)) == _lib.EUNSUPPORTED
