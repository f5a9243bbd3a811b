"""fp64 numpy reference of the operator UDE kernels (operator.cuh): du = D1 NN(u) + D2 u.

Each solver runs the kernels' algorithm step for step, one trajectory at a time:
- fixed-step Tsit5 with the interpolating adjoint on the same grid;
- adaptive Tsit5 (OrdinaryDiffEq's PI controller and initial step, saves from the free interpolant) with the replay adjoint
  split at the save times;
- fixed-step RKC2, whose adjoint steps lambda backwards with RKC2 itself over the cubic Hermite interpolant and takes the
  theta-gradient with the recurrence's quadrature weights (the oracle's ude_adjoint_rkc2_fixed).
Gradients come back as (grad_theta, grad_u0) for an explicit cotangent dL/dout[n_save, d], or with the fused L2
sum w (out - data)^2.  Also the transcription of Climate/NeuralPDE/npde.jl (getops, getu0, ode_i)."""
import numpy as np

from forced_ref import TS_A as A, TS_B as B, TS_BT as BTILDE, TS_C as C, interp_w as bw   # the Tsit5 tableau (tsit5.cuh)


ACTS = {0: (lambda z: z, lambda z, h: np.ones_like(z)),
        1: (np.tanh, lambda z, h: 1.0 - h * h),
        2: (lambda z: np.exp(-z * z), lambda z, h: -2.0 * z * h)}


class Model:
    """widths [d, ..., m], acts per layer (0 identity, 1 tanh, 2 rbf), D1 [d, m], D2 [d, d] or None."""

    def __init__(self, widths, acts, D1, D2=None, lossw=None):
        self.widths, self.acts = list(widths), list(acts)
        self.D1 = np.asarray(D1, dtype=np.float64)
        self.D2 = None if D2 is None else np.asarray(D2, dtype=np.float64)
        self.d = widths[0]
        self.P = sum(a * b + b for a, b in zip(widths[:-1], widths[1:]))
        self.lossw = np.ones(self.d) if lossw is None else np.asarray(lossw, dtype=np.float64)

    def layers(self, th):
        out, o = [], 0
        for a, b, k in zip(self.widths[:-1], self.widths[1:], self.acts):
            W = th[o:o + a * b].reshape(a, b).T   # vec(W) column-major
            o += a * b
            out.append((W, th[o:o + b], k, o - a * b))
            o += b
        return out

    def rhs(self, th, u):
        x = u
        for W, b, k, _ in self.layers(th):
            x = ACTS[k][0](W @ x + b)
        f = self.D1 @ x
        return f if self.D2 is None else f + self.D2 @ u

    def vjp(self, th, u, g, w, gth):
        """returns (df/du)^T g; gth += w (df/dtheta)^T g."""
        xs, zs, x = [u], [], u
        L = self.layers(th)
        for W, b, k, _ in L:
            z = W @ x + b
            x = ACTS[k][0](z)
            zs.append(z)
            xs.append(x)
        v = self.D1.T @ g
        for l in range(len(L) - 1, -1, -1):
            W, b, k, o = L[l]
            dl = v * ACTS[k][1](zs[l], xs[l + 1])
            a, bb = W.shape[1], W.shape[0]
            gth[o:o + a * bb] += w * np.outer(xs[l], dl).ravel()   # entry k * b + i = x_k dl_i
            gth[o + a * bb:o + a * bb + bb] += w * dl
            v = W.T @ dl
        return v if self.D2 is None else v + self.D2.T @ g


def _cot(model, out_s, c, fused):
    """(lambda jump, loss) of one save: c is dL/dout, or the data with the fused L2."""
    if fused:
        r = out_s - c
        return 2.0 * model.lossw * r, float(np.sum(model.lossw * r * r))
    return c, 0.0


# ---------------------------------------------------------------- Tsit5, fixed step
def tsit5_fixed(model, th, u0, t0, dt, n_steps, save_every=1):
    u = np.array(u0, dtype=np.float64)
    k = [None] * 7
    k[0] = model.rhs(th, u)
    out, ustep, dense = [u.copy()], [u.copy()], [[None] * 7 for _ in range(n_steps)]
    for s in range(n_steps):
        for i in range(1, 7):
            g = u + dt * sum(A[i, j] * k[j] for j in range(i))
            if i == 6:
                un = g
            k[i] = model.rhs(th, g)
        dense[s] = list(k)
        u = un
        ustep.append(u.copy())
        if (s + 1) % save_every == 0:
            out.append(u.copy())
        k[0] = k[6]
    return np.array(out), (np.array(ustep), dense)


def tsit5_fixed_adjoint(model, th, rec, dt, n_steps, save_every, cot, fused=False):
    ustep, dense = rec
    gth = np.zeros(model.P)
    n_save = n_steps // save_every + 1
    lam, loss = _cot(model, ustep[n_steps], cot[n_save - 1], fused)
    lam = lam.copy()
    bws = [bw(1.0 - C[i]) for i in range(6)]
    for s in range(n_steps - 1, -1, -1):
        kl = [None] * 6
        for i in range(6):
            x = ustep[s] + dt * sum(bws[i][j] * dense[s][j] for j in range(7))
            g = lam + dt * sum(A[i, j] * kl[j] for j in range(i))
            kl[i] = model.vjp(th, x, g, dt * B[i], gth)
        lam = lam + dt * sum(B[j] * kl[j] for j in range(6))
        if s % save_every == 0:
            j, l = _cot(model, ustep[s], cot[s // save_every], fused)
            lam = lam + j
            loss += l
    return gth, lam, loss


# ---------------------------------------------------------------- Tsit5, adaptive
def tsit5_adaptive(model, th, u0, t0, save_dt, n_save, abstol, reltol, max_steps=100000):
    """returns out [n_save, d], record (steps: list of (t, h, u, k[7])), status (0 ok, 1 non-finite, 2 max_steps)."""
    d = model.d
    t1 = t0 + save_dt * (n_save - 1)
    clip = 1e-12
    u = np.array(u0, dtype=np.float64)
    k = [None] * 7
    k[0] = model.rhs(th, u)
    out = np.full((n_save, d), np.nan)
    out[0] = u
    sk = abstol + reltol * np.abs(u)
    d0 = np.sqrt(np.sum((u / sk) ** 2) / d)
    d1 = np.sqrt(np.sum((k[0] / sk) ** 2) / d)
    dt0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    dt0 = min(dt0, t1 - t0)
    f1 = model.rhs(th, u + dt0 * k[0])
    d2 = np.sqrt(np.sum(((f1 - k[0]) / sk) ** 2) / d) / dt0
    dm = max(d1, d2)
    dt1 = max(1e-6, dt0 * 1e-3) if dm <= 1e-15 else 10.0 ** (-(2.0 + np.log10(dm)) / 5.0)
    dt = min(100 * dt0, dt1, t1 - t0)
    t, qold, isave, steps, status = t0, 1e-4, 1, [], 0
    while isave < n_save:
        h, clipped = dt, False
        if t + h >= t1 - clip * abs(t1):
            h, clipped = t1 - t, True
        for i in range(1, 7):
            g = u + h * sum(A[i, j] * k[j] for j in range(i))
            if i == 6:
                un = g
            k[i] = model.rhs(th, g)
        e = h * sum(BTILDE[j] * k[j] for j in range(7))
        sc = abstol + reltol * np.maximum(np.abs(u), np.abs(un))
        EEst = np.sqrt(np.sum((e / sc) ** 2) / d)
        if not EEst <= 1e300:
            status = 1
            break
        q11 = EEst ** 0.14
        q = min(max(q11 / qold ** 0.08 / 0.9, 0.1), 5.0)
        if EEst <= 1.0:
            if len(steps) >= max_steps:
                status = 2
                break
            tn = t1 if clipped else t + h
            steps.append((t, h, u.copy(), list(k)))
            while isave < n_save:
                ts = t0 + save_dt * isave
                if ts > tn + clip * abs(tn):
                    break
                out[isave] = u + h * sum(b * kk for b, kk in zip(bw(min((ts - t) / h, 1.0)), k))
                isave += 1
            qold = max(EEst, 1e-4)
            dt = h / q if (not clipped or h >= dt) else max(dt, h / q)
            t = tn
            u = un
            k[0] = k[6]
        else:
            dt = h / min(5.0, q11 / 0.9)
    if status == 0 and not np.all(np.isfinite(u)):
        status = 1
    return out, (steps, t), status


def tsit5_adaptive_adjoint(model, th, rec, t0, save_dt, n_save, out, cot, fused=False):
    steps, tend = rec
    eta = 1e-10
    gth = np.zeros(model.P)
    isave = n_save - 1
    lam, loss = _cot(model, out[isave], cot[isave], fused)
    lam = lam.copy()
    isave -= 1
    tgrid = [s[0] for s in steps] + [tend]
    for s in range(len(steps) - 1, -1, -1):
        tn, tn1 = tgrid[s], tgrid[s + 1]
        hn = tn1 - tn
        eps = eta * hn
        _, _, us, ks = steps[s]
        cur = tn1
        while cur > tn + eps:
            ts = t0 + save_dt * isave
            ta = ts if (isave >= 0 and ts > tn + eps) else tn
            h = cur - ta
            kl = [None] * 6
            for i in range(6):
                Th = min(max((cur - C[i] * h - tn) / hn, 0.0), 1.0)
                x = us + hn * sum(b * kk for b, kk in zip(bw(Th), ks))
                g = lam + h * sum(A[i, j] * kl[j] for j in range(i))
                kl[i] = model.vjp(th, x, g, h * B[i], gth)
            lam = lam + h * sum(B[j] * kl[j] for j in range(6))
            cur = ta
            if isave >= 0 and abs(ts - ta) <= eps:
                j, l = _cot(model, out[isave], cot[isave], fused)
                lam = lam + j
                loss += l
                isave -= 1
    return gth, lam, loss


# ---------------------------------------------------------------- RKC2, fixed step
def rkc2_tables(s):
    """the oracle's recurrence tables (oracle.rkc2_coefficients), as a dict of arrays."""
    from oracle import oracle as O
    return O.rkc2_coefficients(s)


def rkc2_fixed(model, th, u0, dt, n_steps, stages, save_every=1):
    t = rkc2_tables(stages)
    u = np.array(u0, dtype=np.float64)
    out, ustep, fstep = [u.copy()], [], []
    for s in range(n_steps):
        F0 = model.rhs(th, u)
        ustep.append(u.copy())
        fstep.append(F0)
        Y0, Y1 = u, u + t["mt1"] * dt * F0
        for j in range(2, stages + 1):
            F = model.rhs(th, Y1)
            mu, nu, mt, ga = t["mu"][j], t["nu"][j], t["mt"][j], t["ga"][j]
            Y0, Y1 = Y1, (1 - mu - nu) * u + mu * Y1 + nu * Y0 + mt * dt * F + ga * dt * F0
        u = Y1
        if (s + 1) % save_every == 0:
            out.append(u.copy())
    ustep.append(u.copy())
    fstep.append(model.rhs(th, u))
    return np.array(out), (np.array(ustep), np.array(fstep))


def rkc2_adjoint(model, th, rec, dt, n_steps, stages, save_every, cot, fused=False):
    t = rkc2_tables(stages)
    ustep, fstep = rec
    gth = np.zeros(model.P)
    n_save = n_steps // save_every + 1
    lam, loss = _cot(model, ustep[n_steps], cot[n_save - 1], fused)
    lam = lam.copy()
    for n in range(n_steps - 1, -1, -1):
        y0, y1, f0, f1 = ustep[n], ustep[n + 1], fstep[n], fstep[n + 1]
        Y0 = Y1 = F0 = None
        for j in range(stages):
            Th = 1.0 - t["c"][j]
            x = (1 - Th) * y0 + Th * y1 + Th * (Th - 1) * ((1 - 2 * Th) * (y1 - y0) + (Th - 1) * dt * f0 + Th * dt * f1)
            F = model.vjp(th, x, lam if j == 0 else Y1, dt * t["w"][j], gth)
            if j == 0:
                F0, Y0, Y1 = F, lam, lam + t["mt1"] * dt * F
            else:
                mu, nu, mt, ga = t["mu"][j + 1], t["nu"][j + 1], t["mt"][j + 1], t["ga"][j + 1]
                Y0, Y1 = Y1, (1 - mu - nu) * lam + mu * Y1 + nu * Y0 + mt * dt * F + ga * dt * F0
        lam = Y1
        if n % save_every == 0:
            j, l = _cot(model, ustep[n], cot[n // save_every], fused)
            lam = lam + j
            loss += l
    return gth, lam, loss


# ---------------------------------------------------------------- Climate/NeuralPDE/npde.jl
def npde_grid(N=32):
    return np.linspace(0.0, 1.0, N)


def npde_ops(N=32, kappa=0.05):
    """getops (npde.jl:17-46): D1 = (1/dz) first difference, D2 = (kappa/dz^2) second difference on the N - 2 interior points
    (the boundary columns drop out through QQ)."""
    n = N - 2
    dz = 1.0 / (N - 1)
    D1 = (np.eye(n) - np.eye(n, k=-1)) / dz
    D2 = kappa / dz ** 2 * (-2.0 * np.eye(n) + np.eye(n, k=1) + np.eye(n, k=-1))
    return D1, D2


def npde_u0(N=32):
    z = npde_grid(N)[1:N - 1]
    return np.exp(-200.0 * (z - 0.75) ** 2)


def npde_phi(u):
    """the known closure of ode_i (npde.jl:54-57)."""
    return np.cos(np.sin(u ** 3) + np.sin(np.cos(u ** 2)))


def npde_truth(saveat, N=32, rtol=1e-10, atol=1e-12):
    """ground_truth (npde.jl:59-63): ode_i solved tightly (scipy Radau stands in for ROCK4 at 1e-9), at saveat -> [len, N - 2]."""
    from scipy.integrate import solve_ivp
    D1, D2 = npde_ops(N)
    sol = solve_ivp(lambda t, u: D1 @ npde_phi(u) + D2 @ u, (saveat[0], saveat[-1]), npde_u0(N), method="Radau",
                    t_eval=saveat, rtol=rtol, atol=atol, jac=lambda t, u: D1 @ np.diag(_dphi(u)) + D2)
    return sol.y.T


def _dphi(u):
    a = np.sin(u ** 3) + np.sin(np.cos(u ** 2))
    da = np.cos(u ** 3) * 3 * u ** 2 + np.cos(np.cos(u ** 2)) * (-np.sin(u ** 2)) * 2 * u
    return -np.sin(a) * da


def glorot(widths, rng):
    """Flux's default Dense init: W ~ U(+-sqrt(6 / (in + out))), b = 0; theta = per layer vec(W) then b."""
    th = []
    for a, b in zip(widths[:-1], widths[1:]):
        lim = np.sqrt(6.0 / (a + b))
        th.append(rng.uniform(-lim, lim, size=(b, a)).T.ravel())   # vec(W) of W [b, a]
        th.append(np.zeros(b))
    return np.concatenate(th)
