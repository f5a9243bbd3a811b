"""Reference Vern7 with its lazy 7th-order dense output (B200UDE_FLAG_VERN7_DENSE), in fp64 numpy on top of the CPU oracle's
right-hand side and its VJP -- the algorithms of csrc/vern7_dense.cuh, written out plainly.

The constants come straight from the 198-double Vern7 block OrdinaryDiffEq 6.19.2 serialized into the reference's
Scenario_1_recovery_0.005.jld2 (committed as golden["scenario_1"]["vern7_consts"]; SURVEY.md App. A.3):
     0..6    c2..c8                    7..49   nonzero a_ij row by row, b1, b4..b9     50..57  bt1, bt4..bt10
    58/59..65    c11 = 1, a_11,j  j in {1, 4..9}
    66/67..74    c12, a_12,j      j in {1, 4..9, 11}
    75/76..84    c13, a_13,j      j in {1, 4..9, 11, 12}
    85/86..95, 96/97..106, 107/108..117   c14..c16, a_i,j  j in {1, 4..9, 11, 12, 13}
    118..124     b_1(theta): coefficients of theta^1..theta^7
    125..160     b_4..b_9: theta^2..theta^7, six each          161..196  b_11..b_16: the same        197  padding
(stages 1-based here, 0-based in the arrays below).

- `dense_record`: adaptive Vern7 (PI controller of the oracle's / kernels' Vern7), steps clipped at the end of tspan only, saveat
  from the interpolant (a save time on a step end takes the step-end state); records tgrid, ustep, hstep.
- `fixed_record`: fixed-step Vern7 with the same record.
- `replay_adjoint`: the kernels' interpolating adjoint -- the accepted steps backwards, each split at the save times inside it,
  lambda stepped with Vern7's 9 update stages, u(t) from the step's interpolant.
- `backward_solve`: a reference-style error-controlled backward Vern7 solve of [lambda; mu] (what DiffEqSensitivity's
  InterpolatingAdjoint does), save times as tstops, u(t) from the forward's interpolant.
"""
import os

import numpy as np

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scenario_1.npz")
UPDATE = [0, 3, 4, 5, 6, 7, 8]                    # stages with b != 0
WEIGHTED = [0, 3, 4, 5, 6, 7, 8, 10, 11, 12, 13, 14, 15]
_EXTRA_COLS = {10: [0, 3, 4, 5, 6, 7, 8], 11: [0, 3, 4, 5, 6, 7, 8, 10], 12: [0, 3, 4, 5, 6, 7, 8, 10, 11],
               13: [0, 3, 4, 5, 6, 7, 8, 10, 11, 12], 14: [0, 3, 4, 5, 6, 7, 8, 10, 11, 12], 15: [0, 3, 4, 5, 6, 7, 8, 10, 11, 12]}


def serialized_block():
    return np.load(_GOLDEN)["vern7_consts"]


def tableau(v=None):
    """-> dict(c[16], A[16, 16], b[16], bt[16], R[16, 8]) with b_i(theta) = sum_p R[i, p] theta^p."""
    v = serialized_block() if v is None else v
    c = np.zeros(16)
    c[1:8] = v[0:7]
    c[8] = c[9] = 1.0
    A = np.zeros((16, 16))
    p = 7
    A[1, 0] = v[p]; p += 1
    A[2, 0], A[2, 1] = v[p], v[p + 1]; p += 2
    for i in range(3, 9):
        A[i, 0] = v[p]; p += 1
        for j in range(2, i):
            A[i, j] = v[p]; p += 1
    A[9, 0] = v[p]; p += 1
    for j in range(2, 7):
        A[9, j] = v[p]; p += 1
    b = np.zeros(16)
    b[0] = v[p]; p += 1
    b[3:9] = v[p:p + 6]; p += 6
    bt = np.zeros(16)
    bt[0] = v[p]; p += 1
    bt[3:10] = v[p:p + 7]; p += 7
    assert p == 58
    for i in range(10, 16):
        c[i] = v[p]; p += 1
        for j in _EXTRA_COLS[i]:
            A[i, j] = v[p]; p += 1
    assert p == 118
    R = np.zeros((16, 8))
    R[0, 1:8] = v[118:125]
    p = 125
    for i in WEIGHTED[1:]:
        R[i, 2:8] = v[p:p + 6]; p += 6
    assert p == 197
    return dict(c=c, A=A, b=b, bt=bt, R=R)


T = tableau()


def weights(th):
    """b_i(theta), i = 0..15."""
    return T["R"] @ (float(th) ** np.arange(8))


def stages(O, m, th, u, h, extra=True, n_update=9):
    """k[16, d]: k_0..k_{n_update-1}, then (extra) the extra stages 10..15 (row 9 stays zero unless n_update = 10)."""
    A = T["A"]
    k = np.zeros((16, m.d))
    k[0] = O.rhs(m, th, u)
    for i in range(1, n_update):
        k[i] = O.rhs(m, th, u + h * (A[i, :i] @ k[:i]))
    if extra:
        for i in range(10, 16):
            k[i] = O.rhs(m, th, u + h * (A[i, :i] @ k[:i]))
    return k


def interpolate(u, h, k, th):
    return u + h * (weights(th) @ k)


def _init_dt(O, m, th, u, t0, t1, abstol, reltol):
    f0 = O.rhs(m, th, u)
    sk = abstol + reltol * np.abs(u)
    d0, d1 = np.sqrt(np.mean((u / sk) ** 2)), np.sqrt(np.mean((f0 / sk) ** 2))
    dt0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    dt0 = min(dt0, t1 - t0)
    f1 = O.rhs(m, th, u + dt0 * f0)
    d2 = np.sqrt(np.mean(((f1 - f0) / sk) ** 2)) / dt0
    dm = max(d1, d2)
    dt1 = max(1e-6, dt0 * 1e-3) if dm <= 1e-15 else 10.0 ** (-(2.0 + np.log10(dm)) / 7.0)
    return min(100 * dt0, dt1, t1 - t0)


ETA = 1e-10   # a save time within ETA h of a step end is that step end (the fp64 kernels' margin)


def dense_record(O, m, th, u0, t0, save_dt, n_save, abstol, reltol, max_steps=4096):
    """-> out[n_save, d], rec = dict(tgrid[nacc+1], ustep[nacc+1, d], hstep[nacc])."""
    b, bt = T["b"], T["bt"]
    gamma, qmin, qmax, beta1, beta2 = 0.9, 0.2, 10.0, 7.0 / 70.0, 2.0 / 35.0
    u = np.asarray(u0, np.float64).copy()
    t1 = t0 + save_dt * (n_save - 1)
    dt = _init_dt(O, m, th, u, t0, t1, abstol, reltol)
    out = np.empty((n_save, m.d))
    out[0] = u
    tgrid, ustep, hstep = [t0], [u.copy()], []
    t, qold, isave = t0, 1e-4, 1
    while isave < n_save:
        h, clipped = dt, False
        if t + h >= t1 - 1e-12 * abs(t1):
            h, clipped = t1 - t, True
        k = stages(O, m, th, u, h, extra=False, n_update=10)
        un = u + h * (b @ k)
        err = h * (bt @ k)
        sc = abstol + reltol * np.maximum(np.abs(u), np.abs(un))
        EEst = np.sqrt(np.mean((err / sc) ** 2))
        if not np.isfinite(EEst):
            raise FloatingPointError("non-finite error estimate")
        q11 = EEst ** beta1
        q = min(max(q11 / qold ** beta2 / gamma, 1 / qmax), 1 / qmin)
        if EEst <= 1.0:
            if len(hstep) >= max_steps:
                raise FloatingPointError("max_steps")
            tn = t1 if clipped else t + h
            eps = ETA * (tn - t)
            ke = None
            while isave < n_save:
                ts = t0 + save_dt * isave
                if ts > tn + eps:
                    break
                if ts >= tn - eps:
                    out[isave] = un
                else:
                    if ke is None:
                        ke = stages(O, m, th, u, h)
                    out[isave] = interpolate(u, h, ke, (ts - t) / h)
                isave += 1
            hstep.append(h)
            qold = max(EEst, 1e-4)
            dt = h / q if (not clipped or h >= dt) else max(dt, h / q)
            t = tn
            u = un
            tgrid.append(t)
            ustep.append(u.copy())
        else:
            dt = h / min(1 / qmin, q11 / gamma)
    return out, dict(tgrid=np.array(tgrid), ustep=np.array(ustep), hstep=np.array(hstep))


def fixed_record(O, m, th, u0, t0, dt, n_steps, save_every):
    """Fixed-step Vern7 -> out[n_save, d] (every save_every steps), rec as dense_record's."""
    b = T["b"]
    u = np.asarray(u0, np.float64).copy()
    us = [u.copy()]
    for _ in range(n_steps):
        k = stages(O, m, th, u, dt, extra=False)
        u = u + dt * (b @ k)
        us.append(u.copy())
    us = np.array(us)
    return us[::save_every].copy(), dict(tgrid=t0 + dt * np.arange(n_steps + 1), ustep=us, hstep=np.full(n_steps, dt))


def replay_adjoint(O, m, th, rec, t0, save_dt, n_save, dLdout):
    """The kernels' interpolating adjoint over the record: dLdout[n_save, d] -> grad_theta[P], grad_u0[d]."""
    A, b, c = T["A"], T["b"], T["c"]
    tg, us, hs = rec["tgrid"], rec["ustep"], rec["hstep"]
    lam = np.zeros(m.d)
    gth = np.zeros(len(th))
    isave = n_save - 1
    for s in range(len(hs) - 1, -1, -1):
        tn, tn1, h, u = tg[s], tg[s + 1], hs[s], us[s]
        eps = ETA * (tn1 - tn)
        k = stages(O, m, th, u, h)
        cur = tn1
        while True:
            while isave >= 0 and t0 + save_dt * isave >= cur - eps:
                lam = lam + dLdout[isave]
                isave -= 1
            if not cur > tn + eps:
                break
            ta = tn
            if isave >= 0 and t0 + save_dt * isave > tn + eps:
                ta = t0 + save_dt * isave
            hh = cur - ta
            kl = np.zeros((9, m.d))
            for i in range(9):
                th_i = min(max((cur - c[i] * hh - tn) / h, 0.0), 1.0)
                x = interpolate(u, h, k, th_i)
                g = lam + hh * (A[i, :i] @ kl[:i])
                kl[i], gi = O.rhs_vjp(m, th, x, g)
                gth += hh * b[i] * gi
            lam = lam + hh * (b[:9] @ kl)
            cur = ta
    while isave >= 0:
        lam = lam + dLdout[isave]
        isave -= 1
    return gth, lam


def backward_solve(O, m, th, rec, t0, save_dt, n_save, dLdout, abstol, reltol):
    """Error-controlled backward Vern7 solve of z = [lambda; mu] from t1 to t0 (dz/ds = [J_u^T lambda; J_theta^T lambda], s = -t),
    the save times as tstops where dLdout jumps into lambda, u(t) from the forward's interpolant; error norm over the whole z
    (OrdinaryDiffEq's default norm).  -> grad_theta, grad_u0, number of accepted backward steps."""
    A, b, bt, c = T["A"], T["b"], T["bt"], T["c"]
    tg, us, hs = rec["tgrid"], rec["ustep"], rec["hstep"]
    cache = {}

    def u_at(t):
        s = int(np.clip(np.searchsorted(tg, t, side="right") - 1, 0, len(hs) - 1))
        if s not in cache:
            cache[s] = stages(O, m, th, us[s], hs[s])
        return interpolate(us[s], hs[s], cache[s], min(max((t - tg[s]) / hs[s], 0.0), 1.0))

    P, d = len(th), m.d

    def f(t, z):
        dl, dm = O.rhs_vjp(m, th, u_at(t), z[:d])
        return np.concatenate([dl, dm])

    gamma, qmin, qmax, beta1, beta2 = 0.9, 0.2, 10.0, 7.0 / 70.0, 2.0 / 35.0
    z = np.zeros(d + P)
    z[:d] = dLdout[n_save - 1]
    nacc = 0
    for isave in range(n_save - 1, 0, -1):
        cur, tend = t0 + save_dt * isave, t0 + save_dt * (isave - 1)
        dt, qold = 0.1 * (cur - tend), 1e-4
        while cur > tend + 1e-12 * max(1.0, abs(tend)):
            h, clipped = dt, False
            if cur - h <= tend + 1e-12 * max(1.0, abs(tend)):
                h, clipped = cur - tend, True
            k = np.zeros((10, d + P))
            for i in range(10):
                k[i] = f(cur - c[i] * h, z + h * (A[i, :i] @ k[:i]))
            zn = z + h * (b[:10] @ k)
            err = h * (bt[:10] @ k)
            sc = abstol + reltol * np.maximum(np.abs(z), np.abs(zn))
            EEst = np.sqrt(np.mean((err / sc) ** 2))
            q11 = EEst ** beta1
            q = min(max(q11 / qold ** beta2 / gamma, 1 / qmax), 1 / qmin)
            if EEst <= 1.0:
                z, cur, qold = zn, (tend if clipped else cur - h), max(EEst, 1e-4)
                dt = h / q
                nacc += 1
            else:
                dt = h / min(1 / qmin, q11 / gamma)
        z[:d] += dLdout[isave - 1]
    return z[d:].copy(), z[:d].copy(), nacc
