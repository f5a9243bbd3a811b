"""fp64 numpy reference of the forced neural ODE with a readout network (B200UDE_MODEL_FORCED, csrc/forced.cuh).

    du = f1([u; gamma(t)]),  y = f0([u; gamma(t)]),  gamma_n(t) = sum_j A_jn cos(w_jn t + phi_jn)

The same algorithms as the kernels, step for step: Tsit5 on a fixed grid with the dense record, the interpolating adjoint on that
grid; the PI-controlled Tsit5 (OrdinaryDiffEq's defaults) with saves from the free interpolant and the replay of its accepted
steps.  Rows per save: the d states, then the r readout outputs.  theta = [f0 layers; f1 layers], each vec(W) column-major then b.

Also the FENE-P truth of NonNewtonianFluids/FENEP.jl:7-39: its algebraic equations theta = lambda tau / f_lambda invert in closed
form, which leaves an explicit ODE in (theta11, theta22, theta12), solved here with classical RK4 on a fine grid.
"""
import numpy as np

TS_C = np.array([0.0, 0.161, 0.327, 0.9, 0.9800255409045097, 1.0, 1.0])
TS_A = np.zeros((7, 7))
TS_A[1, 0] = 0.161
TS_A[2, :2] = [-0.008480655492356989, 0.335480655492357]
TS_A[3, :3] = [2.8971530571054935, -6.359448489975075, 4.3622954328695815]
TS_A[4, :4] = [5.325864828439257, -11.748883564062828, 7.4955393428898365, -0.09249506636175525]
TS_A[5, :5] = [5.86145544294642, -12.92096931784711, 8.159367898576159, -0.071584973281401, -0.028269050394068383]
TS_A[6, :6] = [0.09646076681806523, 0.01, 0.4798896504144996, 1.379008574103742, -3.290069515436081, 2.324710524099774]
TS_B = TS_A[6, :6].copy()
TS_BT = np.array([-0.001780011052225777, -0.0008164344596567469, 0.007880878010261995, -0.1447110071732629, 0.5823571654525552,
                  -0.45808210592918697, 0.015151515151515152])
TS_R = np.zeros((7, 5))
TS_R[0, 1:] = [1.0, -2.763706197274826, 2.9132554618219126, -1.0530884977290216]
TS_R[1, 2:] = [0.13169999999999998, -0.2234, 0.1017]
TS_R[2, 2:] = [3.9302962368947516, -5.941033872131505, 2.490627285651253]
TS_R[3, 2:] = [-12.411077166933676, 30.33818863028232, -16.548102889244902]
TS_R[4, 2:] = [37.50931341651104, -88.1789048947664, 47.37952196281928]
TS_R[5, 2:] = [-27.896526289197286, 65.09189467479366, -34.87065786149661]
TS_R[6, 2:] = [1.5, -4.0, 2.5]

ACT = {"identity": 0, "tanh": 1, "rbf": 2}


def interp_w(th):
    """weights of the free 4th-order interpolant at Theta (b_j(Theta))"""
    return np.array([th * (TS_R[j, 1] + th * (TS_R[j, 2] + th * (TS_R[j, 3] + th * TS_R[j, 4]))) for j in range(7)])


class Model:
    """widths0 / acts0: f0 (d+1 -> ... -> r); widths1 / acts1: f1 (d+1 -> ... -> d); acts as 'tanh' / 'identity' / 'rbf'."""

    def __init__(self, widths0, acts0, widths1, acts1, J=1):
        self.w0, self.a0, self.w1, self.a1, self.J = list(widths0), list(acts0), list(widths1), list(acts1), J
        self.D = self.w1[-1]
        self.R = self.w0[-1]
        assert self.w0[0] == self.D + 1 and self.w1[0] == self.D + 1
        self.P0 = sum(a * b + b for a, b in zip(self.w0[:-1], self.w0[1:]))
        self.P = self.P0 + sum(a * b + b for a, b in zip(self.w1[:-1], self.w1[1:]))

    def layers(self, theta, c):
        ws, acts, off = (self.w0, self.a0, 0) if c == 0 else (self.w1, self.a1, self.P0)
        out = []
        for nin, nout, a in zip(ws[:-1], ws[1:], acts):
            W = theta[off:off + nin * nout].reshape(nout, nin, order="F")
            b = theta[off + nin * nout:off + nin * nout + nout]
            out.append((W, b, a, off))
            off += nin * nout + nout
        return out

    # ---- chains, batched over trajectories (x: [nin, N]) ----
    @staticmethod
    def act(a, z):
        return np.tanh(z) if a == "tanh" else (np.exp(-z * z) if a == "rbf" else z)

    def chain(self, theta, c, x):
        h = x
        for W, b, a, _ in self.layers(theta, c):
            h = self.act(a, W @ h + b[:, None])
        return h

    def chain_vjp(self, theta, c, x, dy, g, w):
        """dx = J^T dy; g (gradient vector) += sum_n w_n (dchain/dtheta)^T dy_n"""
        hs, pres = [x], []
        L = self.layers(theta, c)
        for W, b, a, _ in L:
            z = W @ hs[-1] + b[:, None]
            pres.append(z)
            hs.append(self.act(a, z))
        q = dy
        for l in range(len(L) - 1, -1, -1):
            W, b, a, off = L[l]
            z, hh = pres[l], hs[l + 1]
            q = q * (1 - hh * hh if a == "tanh" else (-2 * z * hh if a == "rbf" else 1.0))
            qw = q * w[None, :]
            nin, nout = W.shape[1], W.shape[0]
            g[off:off + nin * nout] += (qw @ hs[l].T).ravel(order="F")
            g[off + nin * nout:off + nin * nout + nout] += qw.sum(axis=1)
            q = W.T @ q
        return q

    # ---- model ----
    def gamma(self, coef, t):
        """coef [3J, N]; t scalar or [N]"""
        g = 0.0
        for j in range(self.J):
            g = coef[3 * j] * np.cos(coef[3 * j + 1] * t + coef[3 * j + 2]) + g
        return g

    def x_of(self, u, gam):
        return np.vstack([u, np.broadcast_to(gam, u.shape[1:])[None, :]])

    def rhs(self, theta, u, gam):
        return self.chain(theta, 1, self.x_of(u, gam))

    def readout(self, theta, u, gam):
        return self.chain(theta, 0, self.x_of(u, gam))

    def rows(self, theta, u, gam):
        return np.vstack([u, self.readout(theta, u, gam)])


# ================================================================ fixed grid
def forward_fixed(m, theta, u0, coef, t0, dt, n_steps, save_every):
    """-> out [n_save, d + r, N], record (ustep [n_steps+1, d, N], dense [6 n_steps + 1, d, N])"""
    u = np.array(u0, dtype=np.float64)
    ustep, dense = [u.copy()], []
    k = [None] * 7
    k[0] = m.rhs(theta, u, m.gamma(coef, t0))
    dense.append(k[0])
    out = [m.rows(theta, u, m.gamma(coef, t0))]
    for s in range(n_steps):
        tn = s * dt + t0
        for i in range(1, 7):
            acc = 0.0
            for j in range(i):
                if TS_A[i, j] != 0.0:
                    acc = TS_A[i, j] * k[j] + acc
            g = dt * acc + u
            if i == 6:
                u = g
            k[i] = m.rhs(theta, g, m.gamma(coef, TS_C[i] * dt + tn))
            dense.append(k[i])
        ustep.append(u.copy())
        if (s + 1) % save_every == 0:
            out.append(m.rows(theta, u, m.gamma(coef, (s + 1) * dt + t0)))
        k[0] = k[6]
    return np.array(out), (np.array(ustep), np.array(dense))


def _save_jump(m, theta, us, gam, cot_rows, fused, lossw, lam, g, lv):
    """cotangent of one save at the state us -> lam (in place), g (in place); returns the loss contribution"""
    D = m.D
    loss = 0.0
    if fused:
        y = m.readout(theta, us, gam)
        r_s = us - cot_rows[:D]
        r_y = y - cot_rows[D:]
        w = lossw[:, None]
        loss = float(((w[:D] * r_s * r_s).sum(axis=0) * lv).sum() + ((w[D:] * r_y * r_y).sum(axis=0) * lv).sum())
        lam += 2 * w[:D] * r_s
        dy = 2 * w[D:] * r_y
    else:
        lam += cot_rows[:D]
        dy = cot_rows[D:]
    dx = m.chain_vjp(theta, 0, m.x_of(us, gam), dy, g, lv)
    lam += dx[:D]
    return loss


def adjoint_fixed(m, theta, rec, coef, t0, dt, n_steps, save_every, cot, fused=False, lossw=None):
    """interpolating adjoint on the fixed grid, as forced::adjoint_kernel.  cot = data (fused) or dL/dout.
    -> loss, grad_theta [P], grad_u0 [d, N]"""
    ustep, dense = rec
    N = ustep.shape[2]
    lossw = np.ones(m.D + m.R) if lossw is None else np.asarray(lossw, np.float64)
    lv = np.ones(N)
    g = np.zeros(m.P)
    lam = np.zeros((m.D, N))
    loss = 0.0
    n_save = n_steps // save_every + 1

    def jump(i):
        nonlocal loss
        row = i * save_every
        loss += _save_jump(m, theta, ustep[row], m.gamma(coef, row * dt + t0), cot[i], fused, lossw, lam, g, lv)

    jump(n_save - 1)
    bw = [interp_w(1.0 - TS_C[i]) for i in range(6)]
    for s in range(n_steps - 1, -1, -1):
        tn1 = (s + 1) * dt + t0
        kl = [None] * 6
        for i in range(6):
            x = dt * sum(bw[i][j] * dense[s * 6 + j] for j in range(7)) + ustep[s]
            a2 = sum((TS_A[i, j] * kl[j] for j in range(i)), np.zeros_like(lam))
            gg = dt * a2 + lam
            kl[i] = m.chain_vjp(theta, 1, m.x_of(x, m.gamma(coef, -TS_C[i] * dt + tn1)), gg, g, dt * TS_B[i] * lv)[:m.D]
        lam = dt * sum(TS_B[j] * kl[j] for j in range(6)) + lam
        if s % save_every == 0:
            jump(s // save_every)
    return loss, g, lam


# ================================================================ adaptive (one trajectory at a time)
def forward_adaptive_one(m, theta, u0, coef, t0, save_dt, n_save, abstol, reltol, max_steps=100000):
    """PI-controlled Tsit5 of one trajectory (u0 [d], coef [3J]), as forced::adaptive_forward_kernel.
    -> out [n_save, d + r], record dict (tgrid, ustep, dense), status"""
    D = m.D
    coef = np.asarray(coef, np.float64)[:, None]
    gam = lambda t: m.gamma(coef, t)  # noqa: E731
    f = lambda u, t: m.rhs(theta, u[:, None], gam(t))[:, 0]  # noqa: E731
    rows = lambda u, t: m.rows(theta, u[:, None], gam(t))[:, 0]  # noqa: E731
    t1 = t0 + save_dt * (n_save - 1)
    gamma_, qmin, qmax, beta1, beta2 = 0.9, 0.2, 10.0, 7 / 50, 2 / 25
    u = np.array(u0, np.float64)
    out = np.full((n_save, D + m.R), np.nan)
    out[0] = rows(u, t0)
    k = [None] * 7
    k[0] = f(u, t0)
    tgrid, ustep, dense = [t0], [u.copy()], [k[0]]
    sk = abstol + reltol * np.abs(u)
    d0 = np.sqrt(np.sum((u / sk) ** 2) / D)
    d1 = np.sqrt(np.sum((k[0] / sk) ** 2) / D)
    dt0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    dt0 = min(dt0, t1 - t0)
    un = f(dt0 * k[0] + u, t0 + dt0)
    d2 = np.sqrt(np.sum(((un - k[0]) / sk) ** 2) / D) / dt0
    dm = max(d1, d2)
    dt1 = max(1e-6, dt0 * 1e-3) if dm <= 1e-15 else 10.0 ** (-(2 + np.log10(dm)) / 5)
    dt = min(100 * dt0, dt1, t1 - t0)
    t, qold, nacc, isave, status = t0, 1e-4, 0, 1, 0
    while isave < n_save:
        h = dt
        clipped = False
        if t + h >= t1 - 1e-12 * abs(t1):
            h, clipped = t1 - t, True
        for i in range(1, 7):
            acc = 0.0
            for j in range(i):
                if TS_A[i, j] != 0.0:
                    acc = TS_A[i, j] * k[j] + acc
            g = h * acc + u
            if i == 6:
                un = g
            k[i] = f(g, TS_C[i] * h + t)
        e = h * sum(TS_BT[j] * k[j] for j in range(7))
        sc = abstol + reltol * np.maximum(np.abs(u), np.abs(un))
        EEst = np.sqrt(np.sum((e / sc) ** 2) / D)
        if not EEst <= 1e300:
            status = 1
            break
        q11 = EEst ** beta1
        q = min(max(q11 / qold ** beta2 / gamma_, 1 / qmax), 1 / qmin)
        if EEst <= 1.0:
            if nacc >= max_steps:
                status = 2
                break
            tn = t1 if clipped else t + h
            dense += [k[i] for i in range(1, 7)]
            while isave < n_save:
                ts = t0 + save_dt * isave
                if ts > tn + 1e-12 * abs(tn):
                    break
                bw = interp_w(min((ts - t) / h, 1.0))
                out[isave] = rows(h * sum(bw[j] * k[j] for j in range(7)) + u, ts)
                isave += 1
            qold = max(EEst, 1e-4)
            dt = h / q if (not clipped or h >= dt) else max(dt, h / q)
            t = tn
            nacc += 1
            tgrid.append(t)
            u = un.copy()
            k[0] = k[6]
            ustep.append(u.copy())
        else:
            dt = h / min(1 / qmin, q11 / gamma_)
    return out, {"tgrid": np.array(tgrid), "ustep": np.array(ustep), "dense": np.array(dense), "nacc": nacc}, status


def adjoint_adaptive_one(m, theta, rec, out, coef, t0, save_dt, n_save, cot, fused=False, lossw=None):
    """replay adjoint of one trajectory's adaptive solve (forced::adaptive_adjoint_kernel): the cotangent of a save taken at the
    saved state `out` [n_save, d + r]; cot [n_save, d + r].  -> loss, grad_theta, grad_u0 [d]"""
    D = m.D
    coef = np.asarray(coef, np.float64)[:, None]
    lossw = np.ones(D + m.R) if lossw is None else np.asarray(lossw, np.float64)
    tg, us_, dn, nacc = rec["tgrid"], rec["ustep"], rec["dense"], rec["nacc"]
    g = np.zeros(m.P)
    lam = np.zeros((D, 1))
    one = np.ones(1)
    loss = 0.0

    def jump(i):
        nonlocal loss
        loss += _save_jump(m, theta, out[i, :D, None], m.gamma(coef, t0 + save_dt * i), cot[i][:, None], fused, lossw, lam, g, one)

    isave = n_save - 1
    jump(isave)
    isave -= 1
    for s in range(nacc - 1, -1, -1):
        tn, tn1 = tg[s], tg[s + 1]
        hn = tn1 - tn
        eps = 1e-10 * hn
        cur = tn1
        while cur > tn + eps:
            ts = t0 + save_dt * isave
            ta = ts if (isave >= 0 and ts > tn + eps) else tn
            h = cur - ta
            kl = [None] * 6
            for i in range(6):
                th = min(max((cur - TS_C[i] * h - tn) / hn, 0.0), 1.0)
                bw = interp_w(th)
                x = hn * sum(bw[j] * dn[s * 6 + j] for j in range(7)) + us_[s]
                a2 = sum((TS_A[i, j] * kl[j] for j in range(i)), np.zeros(D))
                gg = (h * a2 + lam[:, 0])[:, None]
                kl[i] = m.chain_vjp(theta, 1, m.x_of(x[:, None], m.gamma(coef, cur - TS_C[i] * h)), gg, g, h * TS_B[i] * one)[:D, 0]
            lam = (h * sum(TS_B[j] * kl[j] for j in range(6)) + lam[:, 0])[:, None]
            cur = ta
            if isave >= 0 and abs(ts - ta) <= eps:
                jump(isave)
                isave -= 1
    return loss, g, lam[:, 0]


# ================================================================ FENE-P truth (FENEP.jl:7-39)
def fenep_rhs(th, gd, lam=2.0, eta=4.0, L=2.0):
    """d(theta11, theta22, theta12)/dt, with tau recovered in closed form from theta = lam tau / f_lambda"""
    a = L * L / (L * L - 3)
    c = lam / (eta * a)
    Th = th[0] + th[1]
    s = Th * L * L / (lam * (L * L - 3) - c * Th)          # tau11 + tau22
    fl = (L * L + c * s) / (L * L - 3)
    t11, t22, t12 = th[0] * fl / lam, th[1] * fl / lam, th[2] * fl / lam
    return np.array([-t11 + 2 * lam * gd * t12 / fl, -t22, -t12 + lam * gd * t22 / fl + eta / fl * gd]), t12


def fenep_truth(tsave, gamma_fn, substeps=200):
    """sigma_exact = tau12 at tsave (tsave[0] the start, theta(0) = 0), classical RK4 with `substeps` steps per save interval"""
    tsave = np.asarray(tsave, np.float64)
    th = np.zeros(3)
    out = [fenep_rhs(th, gamma_fn(tsave[0]))[1]]
    for a, b in zip(tsave[:-1], tsave[1:]):
        h = (b - a) / substeps
        t = a
        for _ in range(substeps):
            k1 = fenep_rhs(th, gamma_fn(t))[0]
            k2 = fenep_rhs(th + 0.5 * h * k1, gamma_fn(t + 0.5 * h))[0]
            k3 = fenep_rhs(th + 0.5 * h * k2, gamma_fn(t + 0.5 * h))[0]
            k4 = fenep_rhs(th + h * k3, gamma_fn(t + h))[0]
            th = th + h / 6 * (k1 + 2 * k2 + 2 * k3 + k4)
            t += h
        out.append(fenep_rhs(th, gamma_fn(b))[1])
    return np.array(out)
