"""A grid of descriptors and what b200ude_create answers for each.

The grid is the product of a fixed set of chains (the tuned shapes, one runtime-shape chain per model, one shape outside the
envelope, a forced chain and two operator chains) with every dtype, solver, stepping mode, sensitivity algorithm, subset of the
four flags and create-time kernel knob.  The descriptor is validated before the device is probed, so the answer is the same
with and without a GPU: a refusal is its return code and message, and a descriptor that passes validation is recorded as
rc = 0 and an empty message, whether create then returns B200UDE_OK or B200UDE_ENODEVICE.
tools/make_golden_descriptors.py writes the answers to tests/golden/descriptor_outcomes.npz.
"""
import ctypes as C
import hashlib
import itertools
import os

# the kernel-selection knobs b200ude_create reads; each is also run at 0
KNOBS = ("B200UDE_SEIR_TC", "B200UDE_FKPP_TUNED", "B200UDE_SEIR_VERN7_TC", "B200UDE_ADAPTIVE_TC", "B200UDE_FKPP_PACKED")

LV, SEIR, FKPP, NODE, SEIR_NODE, FORCED, OPERATOR = range(7)
SEIR_CONSTS = (10.0, 0.5944, 0.4239, 1117.3, 0.02, 1 / 3, 1 / 5, 0.2, 1 / 11.2)

# name: (model, state_dim, widths, acts, n_prefix, n_suffix, consts)
CHAINS = {
    "lv32": (LV, 2, (2, 32, 32, 2), (1, 1, 0), 0, 0, (1.3, 1.8)),
    "lv5_p0": (LV, 2, (2, 5, 5, 5, 2), (2, 2, 2, 0), 0, 0, (1.3, 1.8)),
    "lv5_p1": (LV, 2, (2, 5, 5, 5, 2), (2, 2, 2, 0), 1, 0, (1.3, 1.8)),
    "lv5_p2": (LV, 2, (2, 5, 5, 5, 2), (2, 2, 2, 0), 2, 0, (1.3, 1.8)),
    "seir64": (SEIR, 7, (3, 64, 64, 1), (1, 1, 0), 0, 0, SEIR_CONSTS),
    "fkpp16_even": (FKPP, 26, (1, 16, 16, 1), (1, 1, 0), 0, 5, ()),
    "fkpp16_odd": (FKPP, 25, (1, 16, 16, 1), (1, 1, 0), 0, 5, ()),
    "lv_shape": (LV, 2, (2, 8, 8, 2), (1, 1, 0), 0, 0, (1.3, 1.8)),
    "seir_shape": (SEIR, 7, (3, 16, 1), (1, 0), 0, 0, SEIR_CONSTS),
    "fkpp_shape": (FKPP, 26, (1, 5, 5, 5, 1), (2, 2, 2, 0), 0, 5, ()),
    "node_shape": (NODE, 3, (3, 16, 3), (1, 0), 0, 0, ()),
    "seir_node_shape": (SEIR_NODE, 7, (7, 16, 7), (1, 0), 0, 0, SEIR_CONSTS),
    "node_too_wide": (NODE, 3, (3, 65, 3), (1, 0), 0, 0, ()),
    "forced": (FORCED, 1, (2, 4, 1, 2, 4, 1), (1, 0, 1, 0), 0, 0, (2, 1)),
    "operator": (OPERATOR, 30, (30, 8, 30), (1, 1), 0, 0, ()),
    "operator_eigen_est": (OPERATOR, 30, (30, 8, 30), (1, 1), 0, 0, (50.0,)),
}


def grid():
    """(key, env knob set to 0 or None, field values) for every descriptor of the grid, in a fixed order."""
    for name, dtype, solver, adaptive, sensealg, flags, knob in itertools.product(
            CHAINS, (0, 1), (0, 1, 2), (0, 1), (0, 1), range(16), (None,) + KNOBS):
        key = f"{name}/dtype{dtype}/solver{solver}/adaptive{adaptive}/sensealg{sensealg}/flags{flags}/{knob or 'defaults'}"
        yield key, knob, dict(dtype=dtype, solver=solver, adaptive=adaptive, sensealg=sensealg, flags=flags, chain=name)


def key_digest(keys):
    """sha256 of the grid's keys in order: the golden file holds the answers of exactly this grid."""
    return hashlib.sha256("\n".join(keys).encode()).hexdigest()


def make_desc(_lib, dtype, solver, adaptive, sensealg, flags, chain):
    model, state_dim, widths, acts, n_prefix, n_suffix, consts = CHAINS[chain]
    d = _lib.Desc()
    d.struct_size = C.sizeof(_lib.Desc)
    d.dtype, d.model, d.state_dim, d.n_layers = dtype, model, state_dim, len(acts)
    for i, w in enumerate(widths):
        d.widths[i] = w
    for i, a in enumerate(acts):
        d.acts[i] = a
    d.n_prefix, d.n_suffix, d.n_consts = n_prefix, n_suffix, len(consts)
    for i, c in enumerate(consts):
        d.consts[i] = c
    d.solver, d.sensealg, d.adaptive, d.flags = solver, sensealg, adaptive, flags
    d.t0, d.dt, d.n_steps, d.save_every = 0.0, 0.1, 10, 2
    d.abstol, d.reltol, d.max_steps, d.n_stages = 1e-6, 1e-3, 64, 8
    d.max_trajectories = 8
    return d


def outcomes(_lib):
    """keys, return codes and messages of the whole grid (0 and "" for a descriptor that passes validation)."""
    L = _lib.lib()
    keys, rcs, msgs = [], [], []
    saved = {k: os.environ.get(k) for k in KNOBS}
    try:
        for key, knob, f in grid():
            for k in KNOBS:
                os.environ.pop(k, None)
            if knob:
                os.environ[knob] = "0"
            d = make_desc(_lib, **f)
            h = C.c_void_p()
            rc = L.b200ude_create(C.byref(d), C.byref(h))
            msg = (L.b200ude_last_error(None) or b"").decode()
            if h.value:
                L.b200ude_destroy(h)
            if rc in (_lib.OK, _lib.ENODEVICE):
                rc, msg = 0, ""
            keys.append(key)
            rcs.append(rc)
            msgs.append(msg)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return keys, rcs, msgs
