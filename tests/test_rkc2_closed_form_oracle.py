"""The closed-form RKC2 reference (rkc2_closed_form.py, mpmath) against the oracle's fp64 recurrence tables at every stage count
2..64, and the closed-form linear solutions against the fp64 references that run the recurrence (CPU only)."""
import os
import sys

import mpmath as mp
import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import operator_ref as R  # noqa: E402
import rkc2_closed_form as CF  # noqa: E402


def recurrence(t, z):
    """one step of the kernels' stage recurrence on y' = z y from y = 1, with the oracle's fp64 tables, carried as the increments
    D_j = Y_j - 1 as the kernels carry them (so that the round-off of the fp64 arithmetic stays below that of the tables)."""
    D0, D1 = np.zeros_like(z), t["mt1"] * z
    for j in range(2, len(t["mu"])):
        mu, nu, mt, ga = t["mu"][j], t["nu"][j], t["mt"][j], t["ga"][j]
        D0, D1 = D1, mu * D1 + nu * D0 + mt * z * (1.0 + D1) + ga * z
    return 1.0 + D1


@pytest.mark.parametrize("s", range(2, 65))
def test_stability_polynomial_beta_and_weights_match_the_oracle_tables(O, s):
    t = O.rkc2_coefficients(s)
    rk = CF.Rkc2(s)
    beta = float(rk.beta)
    assert abs(t["beta"] - beta) <= 1e-12 * beta
    z = np.linspace(-beta, 0.0, 50)
    P = np.array([float(rk.P(v)) for v in z])
    # The table entries are fp64 numbers that multiply z, so rounding them alone moves the polynomial by ~eps |z| (2.7e-13 at the
    # end of the s = 64 interval): the bound is relative to 1 + |z|.  Tables from fp64 recurrences for T_j, T_j', T_j'' (whose
    # error grows like j^2 eps) missed it by 70x at s = 64.
    err = np.abs(recurrence(t, z) - P)
    assert (err <= 2e-15 * (1.0 + np.abs(z))).all(), (err / (1.0 + np.abs(z))).max()
    assert abs(t["w"].sum() - 1.0) <= 1e-13
    zz = np.linspace(-beta, 0.0, 401)
    with mp.workdps(CF.DPS):
        assert all(abs(rk.P(v)) <= 1 for v in zz)


@pytest.mark.parametrize("s", [2, 7, 33])
def test_step_matrix_against_the_recurrence_on_a_matrix(O, s):
    rng = np.random.default_rng(s)
    d = 6
    Q = np.linalg.qr(rng.normal(size=(d, d)))[0]
    hM = Q @ np.diag(-np.geomspace(1e-2, 0.9 * O.rkc2_coefficients(s)["beta"], d)) @ Q.T + 0.01 * rng.normal(size=(d, d))
    t = O.rkc2_coefficients(s)
    Y0, Y1 = np.eye(d), np.eye(d) + t["mt1"] * hM
    for j in range(2, s + 1):
        mu, nu, mt, ga = t["mu"][j], t["nu"][j], t["mt"][j], t["ga"][j]
        Y0, Y1 = Y1, (1 - mu - nu) * np.eye(d) + mu * Y1 + nu * Y0 + mt * hM @ Y1 + ga * hM
    assert np.abs(CF.step_matrix(s, hM) - Y1).max() <= 1e-11
    assert np.abs(CF.step_matrix(s, hM, 3) - Y1 @ Y1 @ Y1).max() <= 1e-11


@pytest.mark.parametrize("s", [2, 9])
def test_linear_operator_solution_and_grad_u0_against_operator_ref(s):
    """the affine closure du = D1 (W u + b) + D2 u through the augmented matrix, against operator_ref's RKC2 (forward and the
    adjoint's dL/du0)."""
    rng = np.random.default_rng(s)
    d, m, h, n, every = 5, 3, 0.05, 12, 3
    D1 = rng.normal(size=(d, m))
    W = 0.3 * rng.normal(size=(m, d))
    b = rng.normal(size=m)
    D2 = -np.diag(rng.uniform(1.0, 0.9 * float(CF.Rkc2(s).beta) / h, d))
    model = R.Model((d, m), (0,), D1, D2)
    theta = np.concatenate([W.T.ravel(), b])
    u0 = rng.normal(size=d)
    cot = rng.normal(size=(n // every + 1, d))
    out, rec = R.rkc2_fixed(model, theta, u0, h, n, s, every)
    _, lam, _ = R.rkc2_adjoint(model, theta, rec, h, n, s, every, cot)
    sol = CF.LinearOperatorSolve(D1, W, b, D2, h, s, n, every)
    assert np.abs(sol.solution(u0) - out).max() <= 1e-12 * np.abs(out).max()
    assert np.abs(sol.grad_u0(cot) - lam).max() <= 1e-12 * np.abs(lam).max()
    assert np.array_equal(CF.linear_operator_solution(D1, W, b, D2, u0, h, s, n, every), sol.solution(u0))


@pytest.mark.parametrize("s", [3, 16])
@pytest.mark.parametrize("w", [(1.0, -2.0, 1.0), (1.0625, -2.0, 0.9375)])
def test_periodic_diffusion_against_the_recurrence_on_the_circulant_matrix(O, s, w):
    nx, n, every = 16, 20, 5
    D0 = 2.25
    beta = O.rkc2_coefficients(s)["beta"]
    h = 0.5 * beta / (4 * D0)
    Mx = D0 * (w[0] * np.roll(np.eye(nx), -1, axis=1) + w[1] * np.eye(nx) + w[2] * np.roll(np.eye(nx), 1, axis=1))
    # row i of Mx picks u_{i-1}, u_i, u_{i+1}
    u = np.random.default_rng(1).normal(size=nx)
    assert np.allclose(Mx @ u, D0 * (w[0] * np.roll(u, 1) + w[1] * u + w[2] * np.roll(u, -1)))
    t = O.rkc2_coefficients(s)
    Y0, Y1 = np.eye(nx), np.eye(nx) + t["mt1"] * h * Mx
    for j in range(2, s + 1):
        mu, nu, mt, ga = t["mu"][j], t["nu"][j], t["mt"][j], t["ga"][j]
        Y0, Y1 = Y1, (1 - mu - nu) * np.eye(nx) + mu * Y1 + nu * Y0 + mt * h * Mx @ Y1 + ga * h * Mx
    ref = np.array([np.linalg.matrix_power(Y1, k) @ u for k in range(0, n + 1, every)])
    got = CF.periodic_diffusion_solution(u, (*w, D0), h, s, n, every)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    cot = np.random.default_rng(2).normal(size=(n // every + 1, nx))
    gref = sum(np.linalg.matrix_power(Y1, k * every).T @ c for k, c in enumerate(cot))
    assert np.abs(CF.periodic_diffusion_grad_u0(cot, (*w, D0), h, s, n, every) - gref).max() <= 1e-12 * np.abs(gref).max()
