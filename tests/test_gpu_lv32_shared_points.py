"""The warp-collective LV 2-32-32-2 adjoint evaluates stage 5 of a backward step and stage 0 of the step below at the one state
they share, u(t_s) = ustep[s]: the chain forward once, the VJP of each stage's lambda argument, and one theta accumulation on
the summed cotangent rows (lv32_wm.cuh).  Checked against the fp64 oracle over the cases of lv32_shared_points.py, and bit for
bit against out, the loss and grad_u0 recorded before the change (tests/golden/lv32_wm_adjoint_bits.json): the shared state is
the same fp32 value the separate evaluations used, so only the order of the theta sums may change."""
import json

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import lv32_shared_points as C  # noqa: E402


@pytest.fixture(autouse=True)
def _warp_collective(monkeypatch):
    monkeypatch.setenv("B200UDE_FWD_WM", "1")
    monkeypatch.setenv("B200UDE_ADJ_WM", "1")


@pytest.mark.parametrize("N,n_steps,save_every", C.CASES)
def test_shared_points_vs_oracle_and_recorded_bits(O, N, n_steps, save_every):
    out, loss, g, gu = C.run(N, n_steps, save_every)
    with open(C.GOLDEN) as f:
        recorded = json.load(f)[C.key(N, n_steps, save_every)]
    assert C.bits_digest(out, loss, gu) == recorded, "out, loss or grad_u0 differ from the recorded bits"

    theta, u0, data = C.inputs(N, n_steps, save_every)
    l64, g64, gu64, out64 = O.ensemble_loss_grad(O.lv_model(), theta.astype(np.float64), u0, data.astype(np.float64), np.ones(2),
                                                 C.DT, n_steps, save_every=save_every, want_out=True)
    e_g = np.linalg.norm(g - g64) / np.linalg.norm(g64)
    e_gu = np.abs(gu - gu64).max() / np.abs(gu64).max()
    print(f"N {N} n_steps {n_steps} save_every {save_every}: grad_theta {e_g:.2e}, grad_u0 {e_gu:.2e}")
    assert np.isfinite(g).all()
    assert np.all(np.abs(out - out64) <= 1e-4 * (1 + np.abs(out64)))
    assert abs(float(loss) - l64) <= 1e-5 * abs(l64)
    # the bounds of test_gpu_parity.py's warp-collective case
    assert e_g <= 2e-5
    assert e_gu <= 2e-5
