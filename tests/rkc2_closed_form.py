"""Closed-form reference of s-stage RKC2 (damping 2/13) on linear problems, in mpmath at 50 digits.

One step of RKC2 on u' = M u multiplies u by the stability polynomial

    P_s(z) = 1 - b_s T_s(w0) + b_s T_s(w0 + w1 z),   w0 = 1 + eps / s^2,  w1 = T_s'(w0) / T_s''(w0),  b_s = T_s''(w0) / T_s'(w0)^2

with real stability interval [-beta(s), 0], beta(s) = (w0 + 1) / w1.  T_s is evaluated from cosh(s acosh x) (valid for every
real or complex x and integer s), its derivatives from the Chebyshev differential equation: nothing here runs the three-term
recurrence that the kernels, the oracle and operator_ref.py run, so these are an independent check of all three.

The adjoint of a linear model steps lambda back with the same recurrence on (df/du)^T = M^T, so a step of the adjoint is
P_s(h M^T) = P_s(h M)^T whatever u the VJP is evaluated at: dL/du0 of a linear solve is closed-form too."""
import mpmath as mp
import numpy as np

DPS = 50
EPS = mp.mpf(2) / 13


def _T(s, x):
    """T_s(x) for real or complex x."""
    return mp.cosh(s * mp.acosh(x))


class Rkc2:
    """the constants of s-stage RKC2 at 50 digits."""

    def __init__(self, s):
        with mp.workdps(DPS):
            self.s = s
            w0 = 1 + EPS / (s * s)
            th = mp.acosh(w0)
            T = mp.cosh(s * th)
            dT = s * mp.sinh(s * th) / mp.sinh(th)
            d2T = (w0 * dT - s * s * T) / (1 - w0 * w0)   # (1 - x^2) T'' - x T' + s^2 T = 0
            self.w0, self.w1 = w0, dT / d2T
            self.b = d2T / (dT * dT)
            self.a = 1 - self.b * T
            self.beta = (w0 + 1) / self.w1

    def P(self, z):
        """P_s(z) at 50 digits: an mpf for real z, an mpc for complex z."""
        with mp.workdps(DPS):
            v = self.a + self.b * _T(self.s, self.w0 + self.w1 * mp.mpc(z))
            return v if isinstance(z, (complex, mp.mpc)) else v.real


def _eig(hM):
    """eigenvalues and eigenvectors of a small dense diagonalisable matrix in mpmath: (E, V, V^-1)."""
    A = mp.matrix(np.asarray(hM, np.float64).tolist())
    E, V = mp.eig(A)
    return E, V, mp.inverse(V)


def _apply(E, V, Vi, fn):
    """V diag(fn(E)) V^-1 as float64 (the real part: hM is real)."""
    X = V * mp.diag([fn(e) for e in E]) * Vi
    return np.array([[float(mp.re(X[i, j])) for j in range(X.cols)] for i in range(X.rows)])


def step_matrix(s, hM, k=1):
    """P_s(hM)^k for a small dense, diagonalisable hM (d <= 65), by eigendecomposition in mpmath: [d, d] float64."""
    r = Rkc2(s)
    with mp.workdps(DPS):
        return _apply(*_eig(hM), lambda e: r.P(mp.mpc(e)) ** k)


def linear_operator_matrix(D1, W, b, D2):
    """the augmented (d + 1)-state matrix of du = D1 (W u + b) + D2 u: z = (u, 1), z' = [[D1 W + D2, D1 b], [0, 0]] z."""
    d = D1.shape[0]
    M = np.zeros((d + 1, d + 1))
    M[:d, :d] = D1 @ W + D2
    M[:d, d] = D1 @ b
    return M


class LinearOperatorSolve:
    """fixed-step RKC2 with s stages on the affine operator closure du = D1 (W u + b) + D2 u (one identity layer), step h,
    n_steps steps, a save every save_every steps; the step map Phi = P_s(h Maug) and its powers computed once in mpmath."""

    def __init__(self, D1, W, b, D2, h, s, n_steps, save_every):
        self.d = D1.shape[0]
        self.n_save = n_steps // save_every + 1
        r = Rkc2(s)
        with mp.workdps(DPS):
            E, V, Vi = _eig(h * linear_operator_matrix(D1, W, b, D2))
            p = [r.P(mp.mpc(e)) for e in E]
            # Phi^(k save_every), k = 0 .. n_save - 1
            self.Phi = [_apply(p, V, Vi, lambda v: v ** (k * save_every)) for k in range(self.n_save)]

    def solution(self, u0):
        """the saved states [n_save, d] from u0 [d]."""
        z0 = np.append(np.asarray(u0, np.float64), 1.0)
        return np.array([(P @ z0)[:self.d] for P in self.Phi])

    def grad_u0(self, cot):
        """dL/du0 [d] of L = sum_k cot[k] . out[k] (cot [n_save, d])."""
        d = self.d
        return sum(P[:d, :d].T @ c for P, c in zip(self.Phi, np.asarray(cot, np.float64)))


def linear_operator_solution(D1, W, b, D2, u0, h, s, n_steps, save_every):
    """the saved states [n_save, d] of fixed-step RKC2 on du = D1 (W u + b) + D2 u."""
    return LinearOperatorSolve(D1, W, b, D2, h, s, n_steps, save_every).solution(u0)


def linear_operator_grad_u0(D1, W, b, D2, cot, h, s, n_steps, save_every):
    """dL/du0 [d] for the cotangents cot [n_save, d] at the saves of the same solve."""
    return LinearOperatorSolve(D1, W, b, D2, h, s, n_steps, save_every).grad_u0(cot)


def stencil_symbol(nx, w1, w2, w3, D0):
    """eigenvalues lambda_k, k = 0 .. nx - 1, of the periodic 3-tap diffusion of the Fisher-KPP model
    (du_i = D0 (w1 u_{i-1} + w2 u_i + w3 u_{i+1}), oracle/ude_oracle_impl.h) on the Fourier mode exp(2 pi i k j / nx)."""
    t = 2 * np.pi * np.arange(nx) / nx
    return D0 * (w1 * np.exp(-1j * t) + w2 + w3 * np.exp(1j * t))


def periodic_diffusion_solution(u0, stencil, h, s, n_steps, save_every):
    """fixed-step RKC2 on the Fisher-KPP model with zero reaction output: the saved states [n_save, nx] from u0 [nx];
    stencil = (w1, w2, w3, D0).  Each Fourier mode k is multiplied by P_s(h lambda_k) per step."""
    u0 = np.asarray(u0, np.float64)
    amp = _mode_factors(len(u0), stencil, h, s, n_steps, save_every)
    U = np.fft.fft(u0)
    return np.array([np.fft.ifft(a * U).real for a in amp])


def periodic_diffusion_grad_u0(cot, stencil, h, s, n_steps, save_every):
    """dL/du0 [nx] of L = sum_k cot[k] . out[k]: the transpose of the stencil has the conjugate symbol."""
    cot = np.asarray(cot, np.float64)
    amp = _mode_factors(cot.shape[1], stencil, h, s, n_steps, save_every)
    return sum(np.fft.ifft(np.conj(a) * np.fft.fft(c)).real for a, c in zip(amp, cot))


def _mode_factors(nx, stencil, h, s, n_steps, save_every):
    """P_s(h lambda_k)^(j save_every) for the saves j: [n_save, nx] complex128."""
    r = Rkc2(s)
    lam = stencil_symbol(nx, *stencil)
    with mp.workdps(DPS):
        p = [r.P(mp.mpc(h * complex(l))) for l in lam]
        return np.array([[complex(v ** (j * save_every)) for v in p] for j in range(n_steps // save_every + 1)])
