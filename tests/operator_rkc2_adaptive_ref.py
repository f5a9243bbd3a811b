"""fp64 numpy reference of adaptive RKC2 on the operator UDE (operator.cuh, kernels 7 and 8), one trajectory at a time.

Forward: each attempt takes the fewest stages s in 2..cap whose real stability interval beta(s) covers 1.05 h rho (none: s = cap
and h = beta(cap) / (1.05 rho)), runs the s-stage RKC2 recurrence, estimates the error with the estimator of Sommeijer, Shampine
and Verwer, est = 0.8 (u_n - u_{n+1}) + 0.4 h (f(u_n) + f(u_{n+1})), and sets the next h with the PI controller of adaptive Tsit5
at order 2 (exponents 7/20, 1/5).  The save times inside a step come from the cubic Hermite interpolant.

Adjoint: the accepted steps replayed backwards, each split at the save times inside it; a piece of length h' runs the RKC2
recurrence of the step's own stage count backwards with u from the step's Hermite interpolant, and the theta-gradient takes
the quadrature weights h' w_j (operator_ref.rkc2_adjoint with dt -> h')."""
import numpy as np

import operator_ref as R
from operator_ref import _cot


def beta(s):
    """length of the real stability interval of s-stage RKC2 (damping 2/13), as b200ude.cu and sciml._rkc2_beta compute it."""
    w0 = 1.0 + (2.0 / 13.0) / (s * s)
    T0, T1, d0, d1, e0, e1 = 1.0, w0, 0.0, 1.0, 0.0, 0.0
    for _ in range(2, s + 1):
        T0, T1, d0, d1, e0, e1 = T1, 2 * w0 * T1 - T0, d1, 2 * T1 + 2 * w0 * d1 - d0, e1, 4 * d1 + 2 * w0 * e1 - e0
    return (w0 + 1.0) * e1 / d1


_TABLES = {}


def tables(s):
    if s not in _TABLES:
        _TABLES[s] = R.rkc2_tables(s)
    return _TABLES[s]


def pick_stages(h, rho, cap):
    """(s, h): the fewest stages s in 2..cap with beta(s) >= 1.05 h rho; none: (cap, beta(cap) / (1.05 rho))."""
    hr = 1.05 * h * rho
    s = 2
    while s < cap and beta(s) < hr:
        s += 1
    if beta(s) < hr:
        return s, beta(s) / (1.05 * rho), True
    return s, h, False


def herm(Th, h, y0, y1, f0, f1):
    return (1 - Th) * y0 + Th * y1 + Th * (Th - 1) * ((1 - 2 * Th) * (y1 - y0) + (Th - 1) * h * f0 + Th * h * f1)


def rkc2_step(model, th, u, F0, h, s):
    t = tables(s)
    Y0, Y1 = u, u + t["mt1"] * h * F0
    for j in range(2, s + 1):
        F = model.rhs(th, Y1)
        mu, nu, mt, ga = t["mu"][j], t["nu"][j], t["mt"][j], t["ga"][j]
        Y0, Y1 = Y1, (1 - mu - nu) * u + mu * Y1 + nu * Y0 + mt * h * F + ga * h * F0
    return Y1


def rkc2_adaptive(model, th, u0, t0, save_dt, n_save, abstol, reltol, rho, cap=64, max_steps=100000, counts=None):
    """returns out [n_save, d], record (ustep [n+1, d], fstep [n+1, d], tgrid [n+1], sstep [n]), status (0 ok, 1 non-finite,
    2 max_steps).  counts, a dict, receives the accepted steps, rejected steps and right-hand sides."""
    d = model.d
    t1 = t0 + save_dt * (n_save - 1)
    clip = 1e-12
    u = np.array(u0, dtype=np.float64)
    F0 = model.rhs(th, u)
    nrhs = 1
    out = np.full((n_save, d), np.nan)
    out[0] = u
    sk = abstol + reltol * np.abs(u)
    d0 = np.sqrt(np.sum((u / sk) ** 2) / d)
    d1 = np.sqrt(np.sum((F0 / sk) ** 2) / d)
    dt0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    dt0 = min(dt0, t1 - t0)
    f1 = model.rhs(th, u + dt0 * F0)
    nrhs += 1
    d2 = np.sqrt(np.sum(((f1 - F0) / sk) ** 2) / d) / dt0
    dm = max(d1, d2)
    dt1 = max(1e-6, dt0 * 1e-3) if dm <= 1e-15 else 10.0 ** (-(2.0 + np.log10(dm)) / 3.0)
    dt = min(100 * dt0, dt1, t1 - t0)
    t, qold, isave, status, nrej = t0, 1e-4, 1, 0, 0
    ustep, fstep, tgrid, sstep = [u.copy()], [F0.copy()], [t0], []
    while isave < n_save:
        h, clipped = dt, False
        if t + h >= t1 - clip * abs(t1):
            h, clipped = t1 - t, True
        s, h, capped = pick_stages(h, rho, cap)
        if capped:
            clipped = False
        un = rkc2_step(model, th, u, F0, h, s)
        F1 = model.rhs(th, un)
        nrhs += s
        est = 0.8 * (u - un) + 0.4 * h * (F0 + F1)
        sc = abstol + reltol * np.maximum(np.abs(u), np.abs(un))
        EEst = np.sqrt(np.sum((est / sc) ** 2) / d)
        if not EEst <= 1e300:
            status = 1
            break
        q11 = EEst ** 0.35
        q = min(max(q11 / qold ** 0.2 / 0.9, 0.1), 5.0)
        if EEst <= 1.0:
            if len(sstep) >= max_steps:
                status = 2
                break
            tn = t1 if clipped else t + h
            while isave < n_save:
                ts = t0 + save_dt * isave
                if ts > tn + clip * abs(tn):
                    break
                out[isave] = herm(min((ts - t) / h, 1.0), h, u, un, F0, F1)
                isave += 1
            qold = max(EEst, 1e-4)
            dt = h / q if (not clipped or h >= dt) else max(dt, h / q)
            t = tn
            u, F0 = un, F1
            ustep.append(u.copy())
            fstep.append(F0.copy())
            tgrid.append(t)
            sstep.append(s)
        else:
            nrej += 1
            dt = h / min(5.0, q11 / 0.9)
    if status == 0 and not np.all(np.isfinite(u)):
        status = 1
    if counts is not None:
        counts.update(accepted=len(sstep), rejected=nrej, rhs=nrhs)
    return out, (np.array(ustep), np.array(fstep), np.array(tgrid), list(sstep)), status


def rkc2_adaptive_adjoint(model, th, rec, t0, save_dt, n_save, out, cot, fused=False):
    """(grad_theta, dL/du0, loss) of the replay adjoint; out are the saved states the forward returned."""
    ustep, fstep, tgrid, sstep = rec
    eta = 1e-10
    gth = np.zeros(model.P)
    isave = n_save - 1
    lam, loss = _cot(model, out[isave], cot[isave], fused)
    lam = lam.copy()
    isave -= 1
    for n in range(len(sstep) - 1, -1, -1):
        tn, tn1 = tgrid[n], tgrid[n + 1]
        hn = tn1 - tn
        eps = eta * hn
        y0, y1, f0, f1 = ustep[n], ustep[n + 1], fstep[n], fstep[n + 1]
        s = sstep[n]
        t = tables(s)
        cur = tn1
        while cur > tn + eps:
            ts = t0 + save_dt * isave
            ta = ts if (isave >= 0 and ts > tn + eps) else tn
            h = cur - ta
            Y0 = Y1 = F0 = None
            for j in range(s):
                Th = min(max((cur - t["c"][j] * h - tn) / hn, 0.0), 1.0)
                x = herm(Th, hn, y0, y1, f0, f1)
                F = model.vjp(th, x, lam if j == 0 else Y1, h * t["w"][j], gth)
                if j == 0:
                    F0, Y0, Y1 = F, lam, lam + t["mt1"] * h * F
                else:
                    mu, nu, mt, ga = t["mu"][j + 1], t["nu"][j + 1], t["mt"][j + 1], t["ga"][j + 1]
                    Y0, Y1 = Y1, (1 - mu - nu) * lam + mu * Y1 + nu * Y0 + mt * h * F + ga * h * F0
            lam = Y1
            cur = ta
            if isave >= 0 and abs(ts - ta) <= eps:
                j, l = _cot(model, out[isave], cot[isave], fused)
                lam = lam + j
                loss += l
                isave -= 1
    return gth, lam, loss
