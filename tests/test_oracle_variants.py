"""The CPU oracle honours the physics constants and the loss weights it is given.

The GPU tests of the kernel variants (tests/test_gpu_kernel_variants.py) compare kernels run with non-default constant tables
and loss weights against the oracle.  That comparison only means something if the oracle itself reads `consts` and `wmask`:
an oracle that fell back to the default tables would agree with a kernel that hard-codes them.  These checks recompute the
right-hand sides in numpy and test the linearity of the weighted loss, without a GPU.
"""
import numpy as np
import pytest

from helpers import glorot_theta


def _mlp(theta, widths, acts, x):
    """The chain in numpy: per layer vec(W) column-major (W is out x in), then b."""
    h, o = np.asarray(x, np.float64), 0
    for nin, nout, a in zip(widths[:-1], widths[1:], acts):
        W = theta[o:o + nin * nout].reshape((nout, nin), order="F")
        b = theta[o + nin * nout:o + nin * nout + nout]
        o += nin * nout + nout
        h = W @ h + b
        h = {"tanh": np.tanh, "rbf": lambda v: np.exp(-v * v), "identity": lambda v: v}[a](h)
    return h


def _theta(widths, seed):
    """Glorot weights and non-zero biases, so that a bias read from the wrong place shows."""
    rng = np.random.default_rng(seed)
    th = glorot_theta(widths, seed).astype(np.float64)
    o = 0
    for nin, nout in zip(widths[:-1], widths[1:]):
        o += nin * nout
        th[o:o + nout] = rng.uniform(-0.5, 0.5, nout)
        o += nout
    return th


@pytest.mark.parametrize("consts", [(0.7, 2.4), (1.3, 1.8), (-0.4, 0.05)])
def test_lv_rhs_reads_the_constants(O, consts):
    widths, acts = (2, 32, 32, 2), ("tanh", "tanh", "identity")
    m = O.lv_model(consts=consts)
    th = _theta(widths, 1)
    for u in ([0.6, 3.1], [1.7, 0.2], [-0.3, 4.4]):
        u = np.asarray(u)
        nn = _mlp(th, widths, acts, u)
        assert np.allclose(O.mlp_forward(m, th, u), nn, rtol=1e-13, atol=1e-14)
        expect = np.array([consts[0] * u[0] + nn[0], -consts[1] * u[1] + nn[1]])
        assert np.allclose(O.rhs(m, th, u), expect, rtol=1e-13, atol=1e-14)


def test_lv5_rhs_constants_and_trainable_rates(O):
    """2-5-5-5-2: with one trainable rate p1 still comes from the constants and p4 from theta[0]; with two both come from theta."""
    widths, acts = (2, 5, 5, 5, 2), ("rbf", "rbf", "tanh", "identity")
    ch = _theta(widths, 2)
    u = np.array([0.8, 2.6])
    nn = _mlp(ch, widths, acts, u)
    m0 = O.lv_model(widths, acts, n_prefix=0, consts=(0.7, 2.4))
    assert np.allclose(O.rhs(m0, ch, u), [0.7 * u[0] + nn[0], -2.4 * u[1] + nn[1]], rtol=1e-13, atol=1e-14)
    m1 = O.lv_model(widths, acts, n_prefix=1, consts=(0.7, 2.4))
    assert np.allclose(O.rhs(m1, np.concatenate([[1.9], ch]), u), [0.7 * u[0] + nn[0], -1.9 * u[1] + nn[1]], rtol=1e-13, atol=1e-14)
    m2 = O.lv_model(widths, acts, n_prefix=2, consts=(0.7, 2.4))
    assert np.allclose(O.rhs(m2, np.concatenate([[1.1, 1.9], ch]), u), [1.1 * u[0] + nn[0], -1.9 * u[1] + nn[1]], rtol=1e-13, atol=1e-14)


SEIR_PERTURB = (0.8, 1.3, 0.7, 1.5, 2.0, 0.6, 1.4, 0.5, 1.7)


def test_seir_rhs_reads_every_constant(O):
    widths, acts = (3, 64, 64, 1), ("tanh", "tanh", "identity")
    for c in (O.SEIR_CONSTS, tuple(a * s for a, s in zip(O.SEIR_CONSTS, SEIR_PERTURB))):
        m = O.make_model(O.MODEL_SEIR, 7, widths, acts, consts=c)
        th = _theta(widths, 3)
        F, b0, _, _, mu, sg, gm, dd, lm = c
        u = np.array([12e6, 40.0, 30.0, 20.0, 14e6, 5.0, 60.0])
        S, E, I, R, N, D, _ = u
        z = _mlp(th, widths, acts, [S / N, I, D / N])[0]
        expect = [-b0 * S * F / N - z - mu * S, b0 * S * F / N + z - (sg + mu) * E, sg * E - (gm + mu) * I, gm * I - mu * R, -mu * N,
                  dd * gm * I - lm * D, sg * E]
        assert np.allclose(O.rhs(m, th, u), expect, rtol=1e-12, atol=1e-9)


def _check_weight_linearity(O, m, theta, u0, y, dt, n_steps, save_every, w):
    d = len(w)
    parts = []
    for c in range(d):
        e = np.zeros(d)
        e[c] = 1.0
        parts.append(O.ensemble_loss_grad(m, theta, u0, y, e, dt, n_steps, save_every=save_every))
    loss, g, gu = O.ensemble_loss_grad(m, theta, u0, y, np.asarray(w, np.float64), dt, n_steps, save_every=save_every)
    l_lin = sum(wc * p[0] for wc, p in zip(w, parts))
    g_lin = sum(wc * p[1] for wc, p in zip(w, parts))
    gu_lin = sum(wc * p[2] for wc, p in zip(w, parts))
    assert abs(loss - l_lin) <= 1e-12 * abs(l_lin)
    assert np.linalg.norm(g - g_lin) <= 1e-12 * np.linalg.norm(g_lin)
    assert np.abs(gu - gu_lin).max() <= 1e-12 * np.abs(gu_lin).max()
    # and the weights matter: the components contribute differently
    assert abs(parts[0][0] - parts[-1][0]) > 1e-3 * abs(l_lin)


@pytest.mark.parametrize("w", [(0.25, 3.0), (0.0, 1.0), (2.0, 0.0)])
def test_lv_loss_is_linear_in_the_weights(O, w):
    from helpers import synthetic_ensemble
    N = 17
    u0, y = synthetic_ensemble(N, seed=2)
    m = O.lv_model(consts=(0.7, 2.4))
    _check_weight_linearity(O, m, _theta((2, 32, 32, 2), 4), u0, y, 0.1, 30, 1, w)


def test_seir_loss_is_linear_in_the_weights(O):
    rng = np.random.default_rng(7)
    widths, acts = (3, 64, 64, 1), ("tanh", "tanh", "identity")
    c = tuple(a * s for a, s in zip(O.SEIR_CONSTS, SEIR_PERTURB))
    m = O.make_model(O.MODEL_SEIR, 7, widths, acts, consts=c)
    N, n_steps, dt, every = 5, 28, 0.25, 4
    u0 = np.zeros((7, N))
    u0[0] = 0.9 * 14e6 * rng.uniform(0.9, 1.0, N)
    u0[1:4] = rng.uniform(0, 50, (3, N)); u0[4] = 14e6; u0[5] = rng.uniform(0, 10, N); u0[6] = rng.uniform(0, 100, N)
    y = rng.uniform(0, 100, (n_steps // every + 1, 7, N))
    _check_weight_linearity(O, m, glorot_theta(widths, seed=2).astype(np.float64), u0, y, dt, n_steps, every, (0.0, 0.5, 2.0, 1.0, 0.0, 0.0, 0.3))
