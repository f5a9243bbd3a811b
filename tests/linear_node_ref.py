"""Closed-form reference for the linear neural ODE du/dt = W u + b (a one-layer identity chain d -> d), independent of every
solver in the project.

With the augmented matrix M = [[W, b], [0, 0]] the solution is [u(t); 1] = expm(M t) [u0; 1].  For the weighted L2 loss
L = sum_i sum_k w_k (u_k(t_i) - y_ik)^2 the exact continuous gradients are
    dL/du0    = sum_i expm(W t_i)^T r_i,                         r_i = 2 w (u(t_i) - y_i)
    dL/dtheta = sum_i r_i . [expm_frechet(M t_i, E_p t_i) [u0; 1]]_{:d}
where E_p is the unit direction of parameter p in the augmented matrix.  theta is laid out as the chains are (FastChain):
vec(W) column-major (W is out x in), then b.
"""
import numpy as np
from scipy.linalg import expm, expm_frechet


def split(theta, d):
    theta = np.asarray(theta, np.float64)
    return theta[:d * d].reshape((d, d), order="F"), theta[d * d:d * d + d]


def augmented(theta, d):
    W, b = split(theta, d)
    M = np.zeros((d + 1, d + 1))
    M[:d, :d], M[:d, d] = W, b
    return M


def solution(theta, u0, ts):
    """u(t_i) for every t in ts -> [len(ts), d]."""
    u0 = np.asarray(u0, np.float64)
    d = len(u0)
    M = augmented(theta, d)
    z0 = np.append(u0, 1.0)
    return np.array([(expm(M * t) @ z0)[:d] for t in ts])


def solution_scalar(a, b, u0, ts):
    """The d = 1 case written out: u(t) = (u0 + b/a) e^{a t} - b/a."""
    ts = np.asarray(ts, np.float64)
    return (u0 + b / a) * np.exp(a * ts) - b / a


def loss_grad(theta, u0, ts, dLdout):
    """Exact gradient of a loss whose cotangent at the save times is dLdout[len(ts), d] -> (grad_theta[d*d + d], grad_u0[d])."""
    u0 = np.asarray(u0, np.float64)
    d = len(u0)
    M = augmented(theta, d)
    z0 = np.append(u0, 1.0)
    P = d * d + d
    gth, gu = np.zeros(P), np.zeros(d)
    for t, r in zip(ts, dLdout):
        if t == 0.0:
            gu += r
            continue
        gu += expm(M[:d, :d] * t).T @ r
        for p in range(P):
            E = np.zeros((d + 1, d + 1))
            if p < d * d:
                E[p % d, p // d] = 1.0          # W[j, i] with p = j + i d (column-major)
            else:
                E[p - d * d, d] = 1.0           # b
            _, dexp = expm_frechet(M * t, E * t)
            gth[p] += r @ (dexp @ z0)[:d]
    return gth, gu


def l2(theta, u0, ts, y, w):
    """(loss, grad_theta, grad_u0, states) of L = sum w (u(t_i) - y_i)^2 for one trajectory (y: [len(ts), d])."""
    out = solution(theta, u0, ts)
    r = np.asarray(w)[None, :] * (out - y)
    g, gu = loss_grad(theta, u0, ts, 2 * r)
    return float((r * (out - y)).sum()), g, gu, out


def observed_orders(hs, errs):
    """Slopes log(e_i / e_{i+1}) / log(h_i / h_{i+1}) of successive refinements."""
    hs, errs = np.asarray(hs, np.float64), np.asarray(errs, np.float64)
    return np.log(errs[:-1] / errs[1:]) / np.log(hs[:-1] / hs[1:])
