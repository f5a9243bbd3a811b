"""The warp-collective adjoint's ensemble dW2 product (lv32_wm.cuh): fp16 2-way split on the words of the other two products,
transposed by movmatrix, with one power-of-two scale per 8/16-trajectory group and one per step in the accumulator.

The cotangents here spread over 2^-20 .. 2^20 inside every group, so the group's scale is set by one row while the others
sit far below it; the default-row tests of test_gpu_parity.py only see rows of similar size."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import glorot_theta, synthetic_ensemble  # noqa: E402

T_SAVE, DT = 30, 0.1
OFF_W2, N_W2 = 2 * 32 + 32, 32 * 32   # theta = [W1 (64), b1 (32), W2 (1024), b2, W3, b3]


def _solver(N, rows, adj_wm, monkeypatch):
    monkeypatch.setenv("B200UDE_FWD_WM", "1")
    monkeypatch.setenv("B200UDE_ADJ_WM", "1" if adj_wm else "0")
    monkeypatch.setenv("B200UDE_WM_R", str(rows))
    monkeypatch.setenv("B200UDE_WM_G", "1")
    import universal_differential_equations_b200 as ude
    chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
    return ude.UDESolver(ude.LotkaVolterraUDE(chain), 0.0, DT, T_SAVE, 1, max_trajectories=N)


def _spread_cotangent(N, seed):
    """dL/dout[n_save, 2, N]: normal entries times 2^k_n, k_n in [-20, 20]; every aligned block of 8 trajectories holds
    both ends of the range"""
    rng = np.random.default_rng(seed)
    k = rng.integers(-20, 21, N)
    k[0::8], k[1::8] = 20, -20
    return (rng.normal(size=(T_SAVE + 1, 2, N)) * np.exp2(k)).astype(np.float32)


def _adjoint(solver, theta, u0, cot):
    solver.set_params(torch.from_numpy(theta.astype(np.float32)).cuda())
    out = solver.forward(torch.from_numpy(u0).cuda())
    g, gu = solver.adjoint(torch.from_numpy(cot).cuda())
    torch.cuda.synchronize()
    return out.cpu().numpy(), g.cpu().numpy(), gu.cpu().numpy()


@pytest.mark.parametrize("rows,N", [(1, 1001), (2, 1001), (2, 4096)])
def test_wm_dw2_spread_cotangent_vs_oracle_and_tc(O, rows, N, monkeypatch):
    theta = glorot_theta((2, 32, 32, 2), seed=4)
    u0, _ = synthetic_ensemble(N, seed=3)
    cot = _spread_cotangent(N, seed=rows)
    s = _solver(N, rows, True, monkeypatch)
    out, g, gu = _adjoint(s, theta, u0, cot)
    s.close()
    s = _solver(N, rows, False, monkeypatch)
    _, g_tc, _ = _adjoint(s, theta, u0, cot)
    s.close()
    # the oracle's L2 gradient with data y = out64 - cot / 2 is the adjoint of the cotangent cot
    m = O.lv_model()
    th64 = theta.astype(np.float64)
    _, _, _, out64 = O.ensemble_loss_grad(m, th64, u0, np.zeros((T_SAVE + 1, 2, N)), np.ones(2), DT, T_SAVE, want_out=True)
    _, g64, gu64 = O.ensemble_loss_grad(m, th64, u0, out64 - 0.5 * cot.astype(np.float64), np.ones(2), DT, T_SAVE)
    assert np.all(np.abs(out - out64) <= 1e-4 * (1 + np.abs(out64)))
    w2, w2_64, w2_tc = (x[OFF_W2:OFF_W2 + N_W2] for x in (g, g64, g_tc))
    e_g = np.linalg.norm(g - g64) / np.linalg.norm(g64)
    e_w2 = np.linalg.norm(w2 - w2_64) / np.linalg.norm(w2_64)
    e_tc = np.linalg.norm(g - g_tc) / np.linalg.norm(g64)
    e_gu = np.abs(gu - gu64).max() / np.abs(gu64).max()
    print(f"rows {rows} N {N}: grad_theta {e_g:.2e}, W2 block {e_w2:.2e}, vs tensor-core family {e_tc:.2e}, grad_u0 {e_gu:.2e}")
    assert np.isfinite(g).all()
    # H100 (400 W power limit): grad_theta 4.1e-7 ... 5.9e-7, W2 block 4.8e-7 ... 6.9e-7, vs tensor-core family 6.7e-7 ... 9.6e-7,
    # grad_u0 5.2e-7 ... 5.6e-7; the bounds are those of test_lv32_warp_collective_variants_vs_oracle
    assert e_g <= 2e-5 and e_w2 <= 2e-5 and e_tc <= 2e-5
    assert e_gu <= 2e-5


@pytest.mark.parametrize("rows", [1, 2])
def test_wm_dw2_deterministic_and_linear(O, rows, monkeypatch):
    """Bitwise repeatable, and exactly linear under a power-of-two scale of the cotangent (every scale in the product is a
    power of two, so doubling the cotangent doubles every intermediate)."""
    N = 2048
    theta = glorot_theta((2, 32, 32, 2), seed=5)
    u0, _ = synthetic_ensemble(N, seed=7)
    cot = _spread_cotangent(N, seed=11)
    s = _solver(N, rows, True, monkeypatch)
    _, g1, gu1 = _adjoint(s, theta, u0, cot)
    _, g2, gu2 = _adjoint(s, theta, u0, cot)
    _, g3, gu3 = _adjoint(s, theta, u0, 2.0 * cot)
    s.close()
    assert np.array_equal(g1, g2) and np.array_equal(gu1, gu2)
    assert np.array_equal(g3, 2.0 * g1) and np.array_equal(gu3, 2.0 * gu1)
