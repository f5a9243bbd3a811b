"""B200UDE_FLAG_CHECKPOINT without a GPU: which descriptors take the checkpointed record of adaptive Tsit5 on the Fisher-KPP UPDE
(InterpolatingAdjoint(checkpointing = true)), and the flag's value in the header and its Python and Julia mirrors."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

RBF = ((1, 5, 5, 5, 1), (2, 2, 2, 0))        # scenario_3.jl's reaction chain
TUNED = ((1, 16, 16, 1), (1, 1, 0))          # the tuned fixed-step chain, routed to the adaptive kernels when adaptive


@pytest.fixture(scope="module")
def nogpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from universal_differential_equations_b200 import _lib
    return _lib


def _desc(_lib, model, dtype=0, widths=RBF[0], acts=RBF[1], state_dim=26, **kw):
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim = dtype, model, state_dim
    d.n_layers = len(acts)
    for i, w in enumerate(widths):
        d.widths[i] = w
    for i, a in enumerate(acts):
        d.acts[i] = a
    d.solver, d.sensealg = _lib.TSIT5, _lib.INTERPOLATING_ADJOINT
    d.t0, d.dt, d.n_steps, d.save_every, d.max_trajectories = 0.0, 0.1, 10, 1, 8
    d.adaptive, d.abstol, d.reltol, d.max_steps = 1, 1e-6, 1e-3, 2048
    if model == _lib.MODEL_FKPP:
        d.n_suffix = 5
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _create(_lib, d):
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.b200ude_create(C.byref(d), C.byref(h))
    if h.value:
        L.b200ude_destroy(h)
    return rc, (L.b200ude_last_error(None) or b"").decode()


@pytest.mark.parametrize("dtype", [0, 1], ids=["fp32", "fp64"])
@pytest.mark.parametrize("Nx", [3, 26, 256])
@pytest.mark.parametrize("chain", [RBF, TUNED], ids=["rbf", "tuned"])
def test_valid_checkpoint_descriptors_reach_the_device_probe(nogpu, dtype, Nx, chain):
    _lib = nogpu
    for flags in (_lib.FLAG_CHECKPOINT, _lib.FLAG_CHECKPOINT | _lib.FLAG_APPROX_TANH, _lib.FLAG_CHECKPOINT | 16):   # other bits: ignored
        d = _desc(_lib, _lib.MODEL_FKPP, dtype, chain[0], chain[1], Nx, flags=flags)
        rc, msg = _create(_lib, d)
        assert rc == _lib.ENODEVICE, (flags, msg)


def _refused(_lib):
    """Descriptors that are valid without the flag (ENODEVICE here) and that the flag makes EUNSUPPORTED."""
    F, V, R, I, D = _lib.MODEL_FKPP, _lib.VERN7, _lib.RKC2, _lib.INTERPOLATING_ADJOINT, _lib.DISCRETE_ADJOINT
    seir = dict(widths=(3, 64, 64, 1), acts=(1, 1, 0), state_dim=7, n_consts=9)
    cases = {
        "fkpp_fixed_step": _desc(_lib, F, adaptive=0, max_steps=0),
        "fkpp16_rkc2_fixed": _desc(_lib, F, widths=TUNED[0], acts=TUNED[1], adaptive=0, solver=R, n_stages=8),
        "fkpp_vern7_discrete_fp32": _desc(_lib, F, solver=V, sensealg=D),
        "fkpp_vern7_discrete_fp64": _desc(_lib, F, 1, solver=V, sensealg=D),
        "lv_adaptive": _desc(_lib, _lib.MODEL_LV, widths=(2, 5, 5, 5, 2), acts=(2, 2, 2, 0), state_dim=2, n_consts=2),
        "lv_fixed_fp64": _desc(_lib, _lib.MODEL_LV, 1, widths=(2, 8, 2), acts=(1, 0), state_dim=2, n_consts=2, adaptive=0),
        "lv_discrete": _desc(_lib, _lib.MODEL_LV, widths=(2, 5, 5, 5, 2), acts=(2, 2, 2, 0), state_dim=2, n_consts=2, adaptive=0,
                             sensealg=D),
        "seir_adaptive": _desc(_lib, _lib.MODEL_SEIR, **seir),
        "seir_vern7_discrete": _desc(_lib, _lib.MODEL_SEIR, 1, solver=V, sensealg=D, **seir),
        "node_adaptive": _desc(_lib, _lib.MODEL_NODE, widths=(3, 16, 3), acts=(1, 0), state_dim=3),
        "node_discrete_fp64": _desc(_lib, _lib.MODEL_NODE, 1, widths=(3, 16, 3), acts=(1, 0), state_dim=3, adaptive=0, sensealg=D),
        "operator_adaptive": _desc(_lib, _lib.MODEL_OPERATOR, widths=(30, 8, 30), acts=(1, 1), state_dim=30),
        "operator_fixed_fp64": _desc(_lib, _lib.MODEL_OPERATOR, 1, widths=(30, 8, 30), acts=(1, 1), state_dim=30, adaptive=0),
        "forced_adaptive": _desc(_lib, _lib.MODEL_FORCED, widths=(2, 4, 1, 2, 4, 1), acts=(1, 0, 1, 0), state_dim=1, n_consts=2),
    }
    cases["forced_adaptive"].consts[0], cases["forced_adaptive"].consts[1] = 2, 1
    for name in ("lv_adaptive", "lv_fixed_fp64", "lv_discrete"):
        cases[name].consts[0], cases[name].consts[1] = 1.3, 1.8
    for name in ("seir_adaptive", "seir_vern7_discrete"):
        for i, c in enumerate((10.0, 0.5944, 0.4239, 1117.3, 0.02, 1 / 3, 1 / 5, 0.2, 1 / 11.2)):
            cases[name].consts[i] = c
    return cases


def test_flag_refused_everywhere_else(nogpu):
    _lib = nogpu
    for name, d in _refused(_lib).items():
        rc, msg = _create(_lib, d)
        assert rc == _lib.ENODEVICE, (name, "the descriptor must be valid without the flag", msg)
        d.flags = _lib.FLAG_CHECKPOINT
        rc, msg = _create(_lib, d)
        assert rc == _lib.EUNSUPPORTED and "B200UDE_FLAG_CHECKPOINT" in msg, (name, rc, msg)


def test_flag_value_agrees_across_header_python_and_julia():
    from universal_differential_equations_b200 import _lib
    with open(os.path.join(ROOT, "include", "b200ude.h")) as f:
        h = int(re.search(r"#define B200UDE_FLAG_CHECKPOINT (\d+)u", f.read()).group(1))
    with open(os.path.join(ROOT, "julia", "B200UDE.jl")) as f:
        jl = int(re.search(r"const FLAG_CHECKPOINT = UInt32\((\d+)\)", f.read()).group(1))
    assert h == _lib.FLAG_CHECKPOINT == jl == 8
    for other in (_lib.FLAG_APPROX_TANH, _lib.FLAG_VERN7_DENSE, _lib.FLAG_DISCRETE_DENSE):
        assert other & _lib.FLAG_CHECKPOINT == 0


@pytest.mark.parametrize("sensealg,approx,bit", [(None, False, 0), ("default", True, 0), ("ckpt", False, 8), ("ckpt", True, 8),
                                                 ("explicit_false", False, 0)])
def test_interpolating_adjoint_checkpointing_sets_the_flag(monkeypatch, sensealg, approx, bit):
    """The descriptor UDESolver hands to b200ude_create, captured by a stand-in library (no device involved)."""
    import universal_differential_equations_b200 as ude
    from universal_differential_equations_b200 import _lib, sciml

    seen = []

    class FakeLib:
        def b200ude_create(self, d, h):
            seen.append(int(d._obj.flags))
            return _lib.EUNSUPPORTED

        def b200ude_last_error(self, h):
            return b"captured"

    monkeypatch.setattr(sciml.torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(sciml.torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(_lib, "lib", lambda: FakeLib())
    sa = {None: None, "default": ude.InterpolatingAdjoint(), "ckpt": ude.InterpolatingAdjoint(autojacvec=ude.ReverseDiffVJP(), checkpointing=True),
          "explicit_false": ude.InterpolatingAdjoint(checkpointing=False)}[sensealg]
    f = ude.FisherKPPUDE(ude.FastChain(ude.FastDense(1, 16, ude.tanh), ude.FastDense(16, 16, ude.tanh), ude.FastDense(16, 1)), 26)
    with pytest.raises(_lib.B200UDEError):
        ude.UDESolver(f, 0.0, 0.5, 10, 1, max_trajectories=4, device="cuda:0", sensealg=sa, approx_tanh=approx, adaptive=True)
    assert seen == [(_lib.FLAG_APPROX_TANH if approx else 0) | bit]
