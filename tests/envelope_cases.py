"""The chain shapes at the edges of the runtime-shape kernels' envelope (1 to 5 dense layers, widths 1 to 64, identity / tanh /
RBF in any layer, NODE state dimension 1 to 8, fp32 theta up to the 12 288-float constant bank), none of them one that
resolve() routes to a tuned kernel, with their inputs.

    id          form          widths                 acts                          P
    node1_lin   NODE d = 1    1-1                    id                            2      one layer, d = 1, closed form
    node8_lin   NODE d = 8    8-8                    id                            72     one layer, MAXD, closed form
    node8_neck  NODE d = 8    8-1-8                  tanh, id                      25     hidden width 1
    lv_mixed5   LV, 1 rate    2-3-64-1-17-2          rbf, tanh, id, rbf, id        401    five layers, identity hidden layer
    lv_bank     LV, 1 rate    2-62-61-64-64-2        tanh x 4, id                  12288  exactly the fp32 constant bank
    lv_bank1    LV, 2 rates   2-62-61-64-64-2        tanh x 4, id                  12289  fp32 refuses, fp64 runs
    node8_max   NODE d = 8    8-64-64-64-64-8        tanh x 4, id                  13576  largest fp64 vector (fp32 refuses)
    seir_1L     SEIR          3-1                    id                            4      one layer on the model-input path

theta is Glorot-uniform times a per-shape factor, with non-zero biases, so that the right-hand side is O(1) over the time span.
"""
import numpy as np

SHAPES = {
    "node1_lin": dict(form="node", widths=(1, 1), acts=("identity",), scale=1.0, fixed=(-1.2, 0.7)),   # du = -1.2 u + 0.7
    "node8_lin": dict(form="node", widths=(8, 8), acts=("identity",), scale=1.0),
    "node8_neck": dict(form="node", widths=(8, 1, 8), acts=("tanh", "identity"), scale=1.0),
    "lv_mixed5": dict(form="lv", rates=1, widths=(2, 3, 64, 1, 17, 2), acts=("rbf", "tanh", "identity", "rbf", "identity"), scale=1.0),
    "lv_bank": dict(form="lv", rates=1, widths=(2, 62, 61, 64, 64, 2), acts=("tanh",) * 4 + ("identity",), scale=1.0),
    "lv_bank1": dict(form="lv", rates=2, widths=(2, 62, 61, 64, 64, 2), acts=("tanh",) * 4 + ("identity",), scale=1.0),
    "node8_max": dict(form="node", widths=(8, 64, 64, 64, 64, 8), acts=("tanh",) * 4 + ("identity",), scale=0.7),
    "seir_1L": dict(form="seir", widths=(3, 1), acts=("identity",), scale=1.0),
}
F32_SHAPES = ["node1_lin", "node8_lin", "node8_neck", "lv_mixed5", "lv_bank", "seir_1L"]
F64_SHAPES = list(SHAPES)
F32_BANK = 12288   # floats of theta the fp32 constant bank holds (b200ude.cu, create)

SEIR_CONSTS = (10.0, 0.5944, 0.4239, 1117.3, 0.02, 1 / 3, 1 / 5, 0.2, 1 / 11.2)


def num_params(name):
    s = SHAPES[name]
    w = s["widths"]
    return s.get("rates", 0) + sum(a * b + b for a, b in zip(w[:-1], w[1:]))


def grid(name):
    """(save_dt, n_save): the saveat grid of the shape's problem."""
    return (0.5, 9) if SHAPES[name]["form"] == "seir" else (0.1, 11)


def theta(name, seed=1):
    s = SHAPES[name]
    if "fixed" in s:
        return np.array(s["fixed"], np.float64)
    rng = np.random.default_rng(seed)
    parts = []
    if s["form"] == "lv":
        parts.append([1.3, 1.7][2 - s["rates"]:])
    for nin, nout in zip(s["widths"][:-1], s["widths"][1:]):
        lim = np.sqrt(6.0 / (nin + nout))
        parts += [s["scale"] * rng.uniform(-lim, lim, nin * nout), rng.uniform(-0.5, 0.5, nout)]
    th = np.concatenate(parts)
    assert len(th) == num_params(name)
    return th


def u0(name, N, seed=0):
    s = SHAPES[name]
    rng = np.random.default_rng(seed)
    if s["form"] == "lv":
        return np.stack([rng.uniform(0.2, 1.0, N), rng.uniform(2.0, 5.0, N)])
    if s["form"] == "seir":
        u = np.tile(np.array([9000.0, 50.0, 100.0, 0.0, 1e4, 5.0, 0.0])[:, None], (1, N))
        u[1:3] *= rng.uniform(0.5, 1.5, (2, N))
        return u
    return rng.uniform(-1.0, 1.0, (s["widths"][0], N))


def oracle_model(O, name):
    s = SHAPES[name]
    if s["form"] == "lv":
        return O.lv_model(s["widths"], s["acts"], n_prefix=s["rates"])
    if s["form"] == "seir":
        return O.make_model(O.MODEL_SEIR, 7, s["widths"], s["acts"], consts=SEIR_CONSTS)
    return O.make_model(O.MODEL_NODE, s["widths"][0], s["widths"], s["acts"])


def ude_form(name):
    import universal_differential_equations_b200 as ude
    s = SHAPES[name]
    w = s["widths"]
    chain = ude.FastChain(*[ude.FastDense(a, b, act) for a, b, act in zip(w[:-1], w[1:], s["acts"])])
    if s["form"] == "lv":
        return ude.LotkaVolterraUDE(chain, trainable_rates=s["rates"])
    if s["form"] == "seir":
        return ude.SEIRExposureUDE(chain)
    return ude.NeuralODE(chain)


def data(O, name, th, u, seed=2):
    """Targets y[n_save, d, N]: the fp64 oracle's fixed-step solution for 0.9 theta plus 5 % noise, so residuals are O(states)."""
    m = oracle_model(O, name)
    sdt, ns = grid(name)
    rng = np.random.default_rng(seed)
    y = np.stack([O.solve_fixed(m, 0.9 * th, u[:, k], sdt / 4, 4 * (ns - 1), save_every=4) for k in range(u.shape[1])], axis=2)
    return y * (1 + 0.05 * rng.standard_normal(y.shape)) + 0.05 * rng.standard_normal(y.shape)
