"""Reference discrete adjoint (ForwardDiffSensitivity's quantity) over an arbitrary recorded step sequence, for the Tsit5 and
Vern7 tableaus, in fp64 numpy on top of the CPU oracle's right-hand side and its VJP.

- `vern7_adaptive_record`: adaptive Vern7 with OrdinaryDiffEq's PI controller and the save times as tstops (the controller of
  the oracle's Vern7 path and of the GPU kernels), recording every accepted step: tgrid, ustep, hstep and which steps end on
  a save point.
- `solve_steps`: the scheme on a given step sequence (frozen steps), for finite differences.
- `adjoint_steps`: the reverse recurrence through the stages of every step,
      kbar_i = h (b_i lambda_{n+1} + sum_{j>i} a_ji gbar_j),  gbar_i = J_u(g_i)^T kbar_i,
      grad_theta += J_theta(g_i)^T kbar_i,  lambda_n = lambda_{n+1} + sum_i gbar_i,
  with the loss cotangent added where a step ends on a save point.  A fixed grid is the special case.
- `torch_loss`: the same scheme in torch fp64 with the step sizes as constants, for autograd.
"""
import numpy as np

TSIT5, VERN7 = 0, 1


def tableau(O, solver):
    """(A, b, S): S = the stages that feed the update (Tsit5: 6 -- k_7 is FSAL; Vern7: 9 -- the 10th is error-only)."""
    if solver == TSIT5:
        c = O.tsit5_constants()
        A = np.zeros((7, 7))
        p = 6
        for i in range(1, 7):
            for j in range(i):
                A[i, j] = c[p]
                p += 1
        bt = c[27:34]
        return A, A[6, :6].copy(), 6, bt
    c = O.vern7_constants()
    A = np.zeros((10, 10))
    p = 7
    A[1, 0] = c[p]; p += 1
    A[2, 0] = c[p]; A[2, 1] = c[p + 1]; p += 2
    for i in range(3, 9):
        A[i, 0] = c[p]; p += 1
        for j in range(2, i):
            A[i, j] = c[p]; p += 1
    A[9, 0] = c[p]; p += 1
    for j in range(2, 7):
        A[9, j] = c[p]; p += 1
    b = np.zeros(10)
    b[0] = c[p]; p += 1
    b[3:9] = c[p:p + 6]; p += 6
    bt = np.zeros(10)
    bt[0] = c[p]; p += 1
    bt[3:10] = c[p:p + 7]
    return A, b, 9, bt


def _stages(O, m, th, A, S, u, h, n_stages=None):
    n_stages = S if n_stages is None else n_stages
    gs, ks = [], []
    for i in range(n_stages):
        g = u + h * sum(A[i, j] * ks[j] for j in range(i) if A[i, j] != 0) if i else u.copy()
        gs.append(g)
        ks.append(O.rhs(m, th, g))
    return gs, ks


def vern7_adaptive_record(O, m, th, u0, t0, save_dt, n_save, abstol, reltol, max_steps=4096):
    """-> out[n_save, d], rec = dict(tgrid[nacc+1], ustep[nacc+1, d], hstep[nacc], save_step[n_save] (step whose end is save
    point i; -1 for t0))."""
    A, b, S, bt = tableau(O, VERN7)
    d = m.d
    gamma, qmin, qmax, beta1, beta2 = 0.9, 0.2, 10.0, 7.0 / 70.0, 2.0 / 35.0
    u = np.asarray(u0, np.float64).copy()
    t1 = t0 + save_dt * (n_save - 1)
    f0 = O.rhs(m, th, u)
    sk = abstol + reltol * np.abs(u)
    d0, d1 = np.sqrt(np.mean((u / sk) ** 2)), np.sqrt(np.mean((f0 / sk) ** 2))
    dt0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    dt0 = min(dt0, t1 - t0)
    f1 = O.rhs(m, th, u + dt0 * f0)
    d2 = np.sqrt(np.mean(((f1 - f0) / sk) ** 2)) / dt0
    dm = max(d1, d2)
    dt1 = max(1e-6, dt0 * 1e-3) if dm <= 1e-15 else 10.0 ** (-(2.0 + np.log10(dm)) / 7.0)
    dt = min(100 * dt0, dt1, t1 - t0)
    out = np.empty((n_save, d))
    out[0] = u
    tgrid, ustep, hstep, save_step = [t0], [u.copy()], [], [-1]
    t, qold, isave = t0, 1e-4, 1
    while isave < n_save:
        tend = t0 + save_dt * isave
        h, clipped = dt, False
        if t + h >= tend - 1e-12 * abs(tend):
            h, clipped = tend - t, True
        gs, ks = _stages(O, m, th, A, S, u, h, n_stages=10)
        un = u + h * sum(b[j] * ks[j] for j in range(10) if b[j] != 0)
        err = h * sum(bt[j] * ks[j] for j in range(10) if bt[j] != 0)
        sc = abstol + reltol * np.maximum(np.abs(u), np.abs(un))
        EEst = np.sqrt(np.mean((err / sc) ** 2))
        if not np.isfinite(EEst):
            raise FloatingPointError("non-finite error estimate")
        q11 = EEst ** beta1
        q = min(max(q11 / qold ** beta2 / gamma, 1 / qmax), 1 / qmin)
        if EEst <= 1.0:
            if len(hstep) >= max_steps:
                raise FloatingPointError("max_steps")
            hstep.append(h)
            if clipped:
                out[isave] = un
                save_step.append(len(hstep) - 1)
                isave += 1
            qold = max(EEst, 1e-4)
            dt = h / q if (not clipped or h >= dt) else max(dt, h / q)
            t = tend if clipped else t + h
            u = un
            tgrid.append(t)
            ustep.append(u.copy())
        else:
            dt = h / min(1 / qmin, q11 / gamma)
    return out, dict(tgrid=np.array(tgrid), ustep=np.array(ustep), hstep=np.array(hstep), save_step=np.array(save_step))


def fixed_record(n_steps, dt, save_every):
    """The record of a fixed grid: every step h = dt, save point i at the end of step i * save_every - 1."""
    return dict(hstep=np.full(n_steps, dt), save_step=np.array([-1] + [i * save_every - 1 for i in range(1, n_steps // save_every + 1)]))


def solve_steps(O, m, th, u0, rec, solver):
    """The scheme on the frozen step sequence rec['hstep'] -> (states at the save points [n_save, d], ustep [steps+1, d])."""
    A, b, S, _ = tableau(O, solver)
    u = np.asarray(u0, np.float64).copy()
    us = [u.copy()]
    for h in rec["hstep"]:
        _, ks = _stages(O, m, th, A, S, u, h)
        u = u + h * sum(b[j] * ks[j] for j in range(S) if b[j] != 0)
        us.append(u.copy())
    us = np.array(us)
    return us[rec["save_step"] + 1], us


def adjoint_steps(O, m, th, ustep, rec, solver, dLdout):
    """Discrete adjoint over the recorded steps: dLdout[n_save, d] -> grad_theta[P], grad_u0[d]."""
    A, b, S, _ = tableau(O, solver)
    hs, save_step = rec["hstep"], rec["save_step"]
    at = {int(s): i for i, s in enumerate(save_step)}
    lam = np.zeros(m.d)
    gth = np.zeros(len(th))
    for n in range(len(hs) - 1, -1, -1):
        if n in at:
            lam = lam + dLdout[at[n]]
        h = hs[n]
        gs, _ = _stages(O, m, th, A, S, ustep[n], h)
        gb = [None] * S
        for i in range(S - 1, -1, -1):
            kb = h * (b[i] * lam + sum((A[j, i] * gb[j] for j in range(i + 1, S) if A[j, i] != 0), np.zeros(m.d)))
            gb[i], g = O.rhs_vjp(m, th, gs[i], kb)
            gth += g
        lam = lam + sum(gb)
    lam = lam + dLdout[0]
    return gth, lam


def torch_loss(O, m, th, u0, rec, solver, y, w):
    """L = sum_i sum_k w_k (u_k(t_i) - y_ik)^2 through a pure-torch scheme on the frozen steps (th, u0: torch fp64 tensors)."""
    import torch
    A, b, S, _ = tableau(O, solver)
    rhs = torch_rhs(m)
    wt = torch.tensor(np.asarray(w, np.float64))
    yt = torch.tensor(np.asarray(y, np.float64))
    at = {int(s): i for i, s in enumerate(rec["save_step"])}
    u = u0
    L = (wt * (u - yt[0]) ** 2).sum()
    for n, h in enumerate(rec["hstep"]):
        ks = []
        for i in range(S):
            g = u + float(h) * sum(float(A[i, j]) * ks[j] for j in range(i) if A[i, j] != 0) if i else u
            ks.append(rhs(th, g))
        u = u + float(h) * sum(float(b[j]) * ks[j] for j in range(S) if b[j] != 0)
        if n in at:
            L = L + (wt * (u - yt[at[n]]) ** 2).sum()
    return L


def torch_rhs(m):
    """The oracle's right-hand side (LV / SEIR / NODE forms) in torch."""
    import torch
    L, widths, acts, pre = m.n_layers, [m.widths[i] for i in range(m.n_layers + 1)], [m.acts[i] for i in range(m.n_layers)], m.n_prefix
    consts = [m.consts[i] for i in range(m.n_consts)]

    def chain(th, x):
        o = pre
        for l in range(L):
            nin, nout = widths[l], widths[l + 1]
            W = th[o:o + nin * nout].reshape(nin, nout).T
            bb = th[o + nin * nout:o + nin * nout + nout]
            o += nin * nout + nout
            a = W @ x + bb
            x = torch.tanh(a) if acts[l] == 1 else (torch.exp(-a * a) if acts[l] == 2 else a)
        return x

    def f(th, u):
        if m.model == 0:   # LV
            a1, a2 = consts[0], consts[1]
            if pre == 1:
                a2 = th[0]
            if pre == 2:
                a1, a2 = th[0], th[1]
            y = chain(th, u)
            return torch.stack([a1 * u[0] + y[0], -a2 * u[1] + y[1]])
        if m.model == 1:   # SEIR
            F, b0, mu, sg, gm, dd, lm = consts[0], consts[1], consts[4], consts[5], consts[6], consts[7], consts[8]
            S_, E, I, R, N, D = u[0], u[1], u[2], u[3], u[4], u[5]
            z = chain(th, torch.stack([S_ / N, I, D / N]))[0]
            inf = b0 * S_ * F / N
            return torch.stack([-inf - z - mu * S_, inf + z - (sg + mu) * E, sg * E - (gm + mu) * I, gm * I - mu * R, -mu * N,
                                dd * gm * I - lm * D, sg * E])
        return chain(th, u)   # NODE
    return f
