"""Adaptive Tsit5 on the Fisher-KPP UPDE (Fisher-KPP-CNN.jl:136 passes no dt): the oracle's replay adjoint, the
reference the GPU kernels are compared against, and the descriptor validation of the new configurations."""
import ctypes as C

import numpy as np
import pytest

from helpers import glorot_theta

SCRIPT = (26, (1, 10, 20, 10, 1), ("tanh", "tanh", "tanh", "identity"))
SMALL = (9, (1, 6, 6, 1), ("tanh", "tanh", "identity"))


def _problem(O, shape, seed=0):
    """theta = [chain | 1.1 -2.5 1.0 | 0 | 6.5] (Fisher-KPP-CNN.jl:100-108), the script's initial pulse, random data."""
    Nx, widths, acts = shape
    m = O.fkpp_model(Nx, widths, acts)
    theta = np.concatenate([glorot_theta(widths, seed=1).astype(np.float64), [1.1, -2.5, 1.0, 0.0, 6.5]])
    assert len(theta) == O.num_params(m)
    x = np.linspace(0.0, 1.0, Nx)
    u0 = 0.5 * (np.tanh((x - 0.4) / 0.02) - np.tanh((x - 0.6) / 0.02))
    ts = np.linspace(0.0, 5.0, 11)
    y = np.random.default_rng(seed).uniform(0.0, 0.5, (len(ts), Nx))
    return m, theta, u0, ts, y


@pytest.mark.parametrize("shape", [SCRIPT, SMALL], ids=["script_26pt", "small_9pt"])
@pytest.mark.parametrize("abstol,reltol,bound", [(1e-6, 1e-3, 1e-5), (1e-8, 1e-6, 1e-8)])
def test_replay_adjoint_matches_error_controlled_backward_solve(O, shape, abstol, reltol, bound):
    m, theta, u0, ts, y = _problem(O, shape)
    out, rec = O.solve_adaptive_dense(m, theta, u0, ts, abstol, reltol)
    assert rec[3] > 10
    dl = 2.0 * (out - y)
    g_rep, gu_rep = O.adjoint_replay(m, theta, ts, rec, dl)
    g_ref, gu_ref, _ = O.adjoint_adaptive(m, theta, ts, rec, dl, abstol, reltol)
    assert np.linalg.norm(g_rep - g_ref) <= bound * np.linalg.norm(g_ref)
    assert np.linalg.norm(gu_rep - gu_ref) <= bound * np.linalg.norm(gu_ref)


@pytest.mark.parametrize("shape", [SCRIPT, SMALL], ids=["script_26pt", "small_9pt"])
def test_replay_gradient_matches_finite_differences(O, shape):
    """Central differences of the adaptive loss at tight tolerances; every stencil weight and D0 checked on its own."""
    m, theta, u0, ts, y = _problem(O, shape)
    tol = 1e-10

    def loss(th):
        out, _ = O.solve_adaptive_dense(m, th, u0, ts, tol, tol, max_steps=20000)
        return ((out - y) ** 2).sum()

    out, rec = O.solve_adaptive_dense(m, theta, u0, ts, tol, tol, max_steps=20000)
    g, _ = O.adjoint_replay(m, theta, ts, rec, 2.0 * (out - y))
    P = len(theta)
    idx = np.arange(P) if P < 120 else np.unique(np.concatenate([np.random.default_rng(2).choice(P - 5, 40, replace=False), np.arange(P - 5, P)]))
    fd = np.empty(len(idx))
    for a, j in enumerate(idx):
        e = np.zeros(P)
        e[j] = 1e-4 * max(1.0, abs(theta[j]))   # large enough that step-sequence changes of the 1e-10 solves stay below 1e-5
        fd[a] = (loss(theta + e) - loss(theta - e)) / (2 * e[j])
    assert np.linalg.norm(g[idx] - fd) <= 1e-4 * np.linalg.norm(fd)
    for j in (P - 5, P - 4, P - 3, P - 1):   # w1, w2, w3, D0
        a = int(np.flatnonzero(idx == j)[0])
        assert abs(g[j] - fd[a]) <= 1e-4 * abs(fd[a]), j
    assert g[P - 2] == 0.0   # the conv bias does not enter the right-hand side


def _fkpp_desc(_lib, dtype, adaptive=1, solver=None, Nx=26):
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim, d.n_layers = dtype, _lib.MODEL_FKPP, Nx, 4
    for i, w in enumerate((1, 10, 20, 10, 1)):
        d.widths[i] = w
    d.acts[0] = d.acts[1] = d.acts[2] = _lib.ACT_TANH
    d.n_suffix = 5
    d.solver = _lib.TSIT5 if solver is None else solver
    d.dt, d.n_steps, d.save_every, d.max_trajectories = 0.5, 10, 1, 8
    d.adaptive, d.abstol, d.reltol, d.max_steps = adaptive, 1e-6, 1e-3, 512
    if solver == _lib.RKC2:
        d.n_stages = 8
    return d


def test_adaptive_fisher_kpp_descriptors_reach_the_device_probe():
    """Without a CUDA device: adaptive Tsit5 Fisher-KPP in fp32 and fp64 is now a valid configuration (ENODEVICE); fixed-step
    fp64 Fisher-KPP and adaptive RKC2 / Vern7 Fisher-KPP stay unsupported."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from universal_differential_equations_b200 import _lib
    L = _lib.lib()
    h = C.c_void_p()
    for dtype in (_lib.F32, _lib.F64):
        assert L.b200ude_create(C.byref(_fkpp_desc(_lib, dtype)), C.byref(h)) == _lib.ENODEVICE and not h.value
    # the tuned 1-16-16-1 reaction chain on a 256-point grid is routed to the runtime-shape adaptive kernels
    d = _fkpp_desc(_lib, _lib.F32, Nx=256)
    d.n_layers = 3
    for i, w in enumerate((1, 16, 16, 1)):
        d.widths[i] = w
    d.acts[2] = _lib.ACT_IDENTITY
    assert L.b200ude_create(C.byref(d), C.byref(h)) == _lib.ENODEVICE
    assert L.b200ude_create(C.byref(_fkpp_desc(_lib, _lib.F64, adaptive=0)), C.byref(h)) == _lib.EUNSUPPORTED
    assert b"adaptive Tsit5" in L.b200ude_last_error(None)
    for dtype in (_lib.F32, _lib.F64):
        for solver in (_lib.RKC2, _lib.VERN7):
            assert L.b200ude_create(C.byref(_fkpp_desc(_lib, dtype, solver=solver)), C.byref(h)) == _lib.EUNSUPPORTED, (dtype, solver)
            assert L.b200ude_create(C.byref(_fkpp_desc(_lib, dtype, adaptive=0, solver=solver)), C.byref(h)) == _lib.EUNSUPPORTED
