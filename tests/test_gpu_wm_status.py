"""Warp-collective LV 2-32-32-2 family: the status word flags a W2 beyond the range of its fp16 operand copy.

The forward product reads W2 scaled by 2 log2(e) (the tanh argument is folded into the staged weights) as fp16 hi/lo pairs,
so |W2| >= 65504 / (2 log2 e) ~ 22 700 makes the copy infinite.  The resulting NaN pre-activations must reach the state
(tanh's clamp keeps a NaN) and be reported per trajectory rather than saturate silently to tanh = +-1.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import glorot_theta, synthetic_ensemble  # noqa: E402

OFF_W2 = 96


@pytest.mark.parametrize("w2,bad", [(2.0e4, False), (3.0e4, True)])
def test_wm_status_reports_fp16_overflow_of_w2(w2, bad, monkeypatch):
    import universal_differential_equations_b200 as ude
    monkeypatch.setenv("B200UDE_FWD_WM", "1")
    monkeypatch.setenv("B200UDE_ADJ_WM", "1")
    chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
    N = 100
    theta = glorot_theta((2, 32, 32, 2), seed=1).astype(np.float32)
    theta[OFF_W2] = w2   # W2[0][0]
    u0, _ = synthetic_ensemble(N)
    solver = ude.UDESolver(ude.LotkaVolterraUDE(chain), 0.0, 0.1, 30, 1, max_trajectories=N)
    solver.set_params(torch.from_numpy(theta).cuda())
    status = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = solver.forward(torch.from_numpy(u0).cuda(), status=status)
    torch.cuda.synchronize()
    st, out = status.cpu().numpy(), out.cpu().numpy()
    if bad:
        assert (st != 0).all()
    else:
        assert (st == 0).all() and np.isfinite(out).all()
    solver.close()
