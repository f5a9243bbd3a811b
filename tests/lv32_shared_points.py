"""Cases of the warp-collective LV 2-32-32-2 adjoint around the step points two backward stages share (lv32_wm.cuh): step
counts 1, 2, 5 and 30 (no shared point, one, several, the benchmark's), saves every 1, 2 or 3 steps where that divides the
step count (a data jump at every shared point or at some of them) and ensembles on both sides of the 8-row / 16-row switch (4224 on 132 SMs) and at the
benchmark's size.  Used by tests/test_gpu_lv32_shared_points.py and tools/make_golden_lv32_adjoint_bits.py."""
import hashlib
import os

import numpy as np

from helpers import glorot_theta, synthetic_ensemble

DT = 0.1
N_STEPS = (1, 2, 5, 30)
SAVE_EVERY = (1, 2, 3)
SIZES = (1, 37, 4224, 4225, 65536)
CASES = [(n, s, e) for n in SIZES for s in N_STEPS for e in SAVE_EVERY if s % e == 0]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lv32_wm_adjoint_bits.json")


def key(N, n_steps, save_every):
    return f"N={N},n_steps={n_steps},save_every={save_every}"


def inputs(N, n_steps, save_every):
    """theta (fp32), u0[2, N], data[n_save, 2, N]: seeded"""
    theta = glorot_theta((2, 32, 32, 2), seed=11).astype(np.float32)
    u0, y = synthetic_ensemble(N, n_steps=n_steps, dt=DT, seed=N + 100 * n_steps)
    return theta, u0, np.ascontiguousarray(y[::save_every][: n_steps // save_every + 1])


def run(N, n_steps, save_every):
    """forward + fused-L2 interpolating adjoint on the warp-collective kernels (B200UDE_FWD_WM = B200UDE_ADJ_WM = 1 must be set
    before the call): out, loss, grad_theta, grad_u0 as numpy fp32"""
    import torch

    import universal_differential_equations_b200 as ude
    theta, u0, data = inputs(N, n_steps, save_every)
    chain = ude.FastChain(ude.FastDense(2, 32, ude.tanh), ude.FastDense(32, 32, ude.tanh), ude.FastDense(32, 2))
    s = ude.UDESolver(ude.LotkaVolterraUDE(chain), 0.0, DT, n_steps, save_every, max_trajectories=N)
    try:
        s.set_params(torch.from_numpy(theta).cuda())
        out = s.forward(torch.from_numpy(u0).cuda())
        loss, g, gu = s.adjoint_l2(torch.from_numpy(data).cuda(), want_grad_u0=True)
        torch.cuda.synchronize()
        return out.cpu().numpy(), loss.cpu().numpy()[0], g.cpu().numpy(), gu.cpu().numpy()
    finally:
        s.close()


def bits_digest(out, loss, grad_u0):
    """sha256 of the bits of out, loss and grad_u0 (lambda at t0): the results the shared points must leave unchanged"""
    h = hashlib.sha256()
    for a in (out, np.asarray(loss, dtype=np.float32), grad_u0):
        h.update(np.ascontiguousarray(a, dtype=np.float32).tobytes())
    return h.hexdigest()
