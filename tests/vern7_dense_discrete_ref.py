"""Reference discrete adjoint (ForwardDiffSensitivity's quantity) of the free-stepping Vern7 solve whose save points come from the
lazy 7th-order interpolant (B200UDE_FLAG_DISCRETE_DENSE), in fp64 numpy over `vern7_dense_ref.dense_record`'s record -- the
algorithm of csrc/vern7_dense_discrete.cuh, written out plainly.

With the accepted step sizes frozen, a save time inside step n at theta = (t_s - t_n) / h_n is
    out_s = u_n + h_n sum_{i in W} b_i(theta) k_i,     W = {0, 3..8, 10..15},
where k_10..k_15 are the extra stages (functions of u_n and k_0..k_8); a save time on a step end is u_{n+1}.

- `save_map`: which step holds each save point, and at which theta (None: on the step end), by the forward's own rule.
- `solve_frozen`: the scheme on the frozen steps with the interpolated saves, for finite differences.
- `adjoint_dense_steps`: the reverse recurrence, stages 15..10 then 8..0 (stage 9 only feeds the error estimate),
      kbar_i = h (b_i lambda_{n+1} [i <= 8] + sum_s b_i(theta_s) sbar_s + sum_{j>i} a_ji gbar_j),  gbar_i = J_u(g_i)^T kbar_i,
      grad_theta += J_theta(g_i)^T kbar_i,  lambda_n = lambda_{n+1} + sum_s sbar_s + sum_i gbar_i.
- `torch_loss`: the same scheme in torch fp64 with the step sizes and thetas as constants, for autograd.
"""
import numpy as np

import vern7_dense_ref as V
from discrete_ref import torch_rhs

A, B = V.T["A"], V.T["b"]
UPDATE_STAGES = list(range(9))
EXTRA_STAGES = list(range(10, 16))


def save_map(rec, t0, save_dt, n_save):
    """-> per step n the list of (save index, theta or None); save point 0 (t0) is in no step."""
    tg = rec["tgrid"]
    per_step = [[] for _ in rec["hstep"]]
    isave = 1
    for n in range(len(per_step)):
        t, tn = tg[n], tg[n + 1]
        eps = V.ETA * (tn - t)
        while isave < n_save:
            ts = t0 + save_dt * isave
            if ts > tn + eps:
                break
            per_step[n].append((isave, None if ts >= tn - eps else (ts - t) / rec["hstep"][n]))
            isave += 1
    assert isave == n_save
    return per_step


def solve_frozen(O, m, th, u0, rec, t0, save_dt, n_save):
    """The scheme on the frozen step sequence rec['hstep'] -> saved states [n_save, d]."""
    u = np.asarray(u0, np.float64).copy()
    out = np.empty((n_save, m.d))
    out[0] = u
    for h, saves in zip(rec["hstep"], save_map(rec, t0, save_dt, n_save)):
        inner = any(theta is not None for _, theta in saves)
        k = V.stages(O, m, th, u, h, extra=inner)
        un = u + h * (B @ k)
        for i, theta in saves:
            out[i] = un if theta is None else V.interpolate(u, h, k, theta)
        u = un
    return out


def adjoint_dense_steps(O, m, th, rec, t0, save_dt, n_save, dLdout):
    """Discrete adjoint over the recorded steps: dLdout[n_save, d] -> grad_theta[P], grad_u0[d]."""
    us, hs = rec["ustep"], rec["hstep"]
    per_step = save_map(rec, t0, save_dt, n_save)
    lam = np.zeros(m.d)
    gth = np.zeros(len(th))
    for n in range(len(hs) - 1, -1, -1):
        u, h = us[n], hs[n]
        sbar_sum = np.zeros(m.d)
        wbar = np.zeros((16, m.d))           # sum_s b_i(theta_s) sbar_s
        for i, theta in per_step[n]:
            if theta is None:
                lam = lam + dLdout[i]
            else:
                sbar_sum += dLdout[i]
                wbar += np.outer(V.weights(theta), dLdout[i])
        inner = any(theta is not None for _, theta in per_step[n])
        k = V.stages(O, m, th, u, h, extra=inner)
        order = (EXTRA_STAGES[::-1] if inner else []) + UPDATE_STAGES[::-1]
        gb = np.zeros((16, m.d))
        for i in order:
            kb = h * (B[i] * lam + wbar[i] + A[i + 1:, i] @ gb[i + 1:])
            gb[i], g = O.rhs_vjp(m, th, u + h * (A[i, :i] @ k[:i]), kb)
            gth += g
        lam = lam + sbar_sum + gb.sum(axis=0)
    lam = lam + dLdout[0]
    return gth, lam


def torch_loss(O, m, th, u0, rec, t0, save_dt, n_save, y, w):
    """L = sum_i sum_k w_k (out_ik - y_ik)^2 through a pure-torch scheme on the frozen steps with the interpolated saves
    (th, u0: torch fp64 tensors)."""
    import torch
    rhs = torch_rhs(m)
    wt = torch.tensor(np.asarray(w, np.float64))
    yt = torch.tensor(np.asarray(y, np.float64))

    def stage(u, h, ks, i):
        return rhs(th, u + h * sum(float(A[i, j]) * ks[j] for j in range(i) if A[i, j] != 0) if i else u)

    u = u0
    L = (wt * (u - yt[0]) ** 2).sum()
    for h, saves in zip(rec["hstep"], save_map(rec, t0, save_dt, n_save)):
        h = float(h)
        ks = {}
        for i in UPDATE_STAGES:
            ks[i] = stage(u, h, ks, i)
        un = u + h * sum(float(B[j]) * ks[j] for j in V.UPDATE)
        if any(theta is not None for _, theta in saves):
            for i in EXTRA_STAGES:
                ks[i] = stage(u, h, ks, i)
        for i, theta in saves:
            if theta is None:
                o = un
            else:
                bw = V.weights(theta)
                o = u + h * sum(float(bw[j]) * ks[j] for j in V.WEIGHTED)
            L = L + (wt * (o - yt[i]) ** 2).sum()
        u = un
    return L
