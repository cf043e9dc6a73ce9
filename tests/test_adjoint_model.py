"""References for the solves with the adjoint (no GPU): z = R^{-H} c and the minimum-norm solution y = Q [z; 0] of A^H y = c, in fp64
(tests/adjoint_oracle.py: np_forwardsolve / np_solve_adj and their complex twins) and in long double (adj_ext), against scipy
and mpmath."""
import numpy as np
import pytest
import scipy.linalg as sla

import adjoint_oracle as AO


def _rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("m,n,k", [(60, 25, 1), (97, 40, 3), (33, 33, 2)])
def test_oracle_adjoint_matches_scipy(oracle, coracle, cplx, m, n, k):
    rng = np.random.default_rng([m, n, k, int(cplx)])
    a = rng.standard_normal((m, n))
    c = rng.standard_normal((n, k))
    if cplx:
        a = a + 1j * rng.standard_normal((m, n))
        c = c + 1j * rng.standard_normal((n, k))
    a = np.asfortranarray(a)
    y_ref = sla.lstsq(a.conj().T, c)[0]                            # minimum-norm solution of A^H y = c (m > n: underdetermined)
    if cplx:
        h, alpha = oracle.np_qr_c(a)
        z64 = np.stack([AO.np_forwardsolve_c(h, alpha, c[:, j]) for j in range(k)], 1)
        y64 = AO.np_solve_adj_c(h, alpha, c)
    else:
        h, alpha = oracle.np_qr(a)
        z64 = np.stack([AO.np_forwardsolve(h, alpha, c[:, j]) for j in range(k)], 1)
        y64 = AO.np_solve_adj(h, alpha, c)
    r = np.triu(h[:n], 1) + np.diag(alpha)
    z_ref = sla.solve_triangular(r, c, trans="C")
    z_ext, y_ext = AO.adj_ext(a, c)
    for z in (z64, z_ext):
        assert _rel(z, z_ref) < 1e-12
    for y in (y64, y_ext):
        assert _rel(y, y_ref) < 1e-12
        assert np.linalg.norm(a.conj().T @ y - c) / (np.linalg.norm(a) * np.linalg.norm(y)) < 1e-14
    # one vector in, one vector out; the long double factorisation is the fp64 one to rounding
    z1, y1 = AO.adj_ext(a, c[:, 0])
    assert z1.shape == (n,) and y1.shape == (m,)
    assert _rel(y1, y_ext[:, 0]) == 0.0


def test_oracle_adjoint_empty_system(coracle):
    a = np.asfortranarray(np.random.default_rng(2).standard_normal((7, 0)))
    z, y = AO.adj_ext(a, np.zeros((0, 2)))
    assert z.shape == (0, 2) and y.shape == (7, 2) and not y.any()


def test_oracle_adjoint_long_double_matches_mpmath(coracle):
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.dps = 50
    m, n = 9, 5
    rng = np.random.default_rng(3)
    a = np.asfortranarray(rng.standard_normal((m, n)))
    c = rng.standard_normal(n)
    _, y_ext = AO.adj_ext(a, c)
    A = mpmath.matrix(a.tolist())
    C = mpmath.matrix(c.tolist())
    # minimum-norm solution of A^T y = c: y = A (A^T A)^{-1} c
    y_mp = A * mpmath.lu_solve(A.T * A, C)
    y_exact = np.array([float(y_mp[i]) for i in range(m)])
    tol = 64 * 2.0 ** -coracle.ext_mant_dig() * np.linalg.cond(a) ** 2 + 2 * np.finfo(float).eps
    assert _rel(y_ext, y_exact) < max(tol, 4 * np.finfo(float).eps)
