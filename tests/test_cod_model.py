"""References for the complete orthogonal decomposition on the pivoted QR (no GPU): the fp64 twin of the device's stages and
the long-double twin of the whole solve (tests/cod_model.py), against numpy.linalg.lstsq, LAPACK dgelsy (scipy) and mpmath."""
import mpmath
import numpy as np
import pytest
import scipy.linalg as sla

import cod_model as CM
import qrcp_model as M


def _rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


def _rank(alpha, rcond=1e-10):
    small = np.nonzero(~(np.abs(alpha) > rcond * abs(alpha[0])))[0]
    return int(small[0]) if small.size else alpha.size


@pytest.mark.parametrize("m,n,r", [(300, 60, 1), (300, 60, 7), (300, 60, 31), (300, 60, 33), (400, 100, 99), (200, 64, 64)])
def test_fp64_twin_matches_lstsq_on_exact_low_rank(coracle, m, n, r):
    A0 = CM.low_rank(m, n, r)
    b = np.random.default_rng([m, n, r]).standard_normal((m, 2))
    fac = M.qrcp_model(A0)[:3]
    assert _rank(fac[1]) == r
    x, F, gamma = CM.cod_fp64(coracle, A0, b, r, fac)
    assert F.shape == (n, r) and gamma.shape == (r,)
    x_np = np.linalg.lstsq(A0, b, rcond=None)[0]
    assert _rel(x, x_np) <= 1e-8
    assert _rel(x, CM.pinv_solve(A0, b, r)) <= 1e-8
    x_ext = CM.cod_ext(A0, fac[2], r, b)
    assert _rel(x, x_ext) <= 1e-10
    if r < n:                                                      # the basic solution has the same residual and a larger norm
        xb = np.zeros((n, 2))
        H, alpha, p = fac
        R11 = M.form_r(H, alpha)[:r, :r]
        for k in range(2):
            c = coracle.apply_qt(np.asfortranarray(H[:, :r]), b[:, k].copy())[:r]
            xb[p[:r], k] = sla.solve_triangular(R11, c)
        for k in range(2):
            assert np.linalg.norm(x[:, k]) < np.linalg.norm(xb[:, k])
            assert abs(np.linalg.norm(A0 @ x[:, k] - b[:, k]) - np.linalg.norm(A0 @ xb[:, k] - b[:, k])) <= 1e-10 * np.linalg.norm(b[:, k])


@pytest.mark.parametrize("m,n,r", [(300, 60, 5), (300, 60, 40), (256, 128, 100)])
def test_fp64_twin_matches_gelsy(coracle, m, n, r):
    A0 = CM.low_rank(m, n, r, noise=1e-13)
    b = np.random.default_rng([m, n, r, 1]).standard_normal(m)
    x_g, _, rank_g, _ = sla.lstsq(A0, b, cond=1e-8, lapack_driver="gelsy")
    assert rank_g == r                                             # gelsy picks the same rank: the answers are comparable
    fac = M.qrcp_model(A0)[:3]
    assert _rank(fac[1], 1e-8) == r
    x = CM.cod_fp64(coracle, A0, b, r, fac)[0]
    assert _rel(x, x_g) <= 1e-8


def _mp_cod(A0, p, r, b):
    """x = P R_r' (R_r R_r')^{-1} (Q'b)[0:r] at 50 digits, from the QR of A[:, p] (sign conventions cancel)."""
    with mpmath.workdps(50):
        m, n = A0.shape
        Ap = mpmath.matrix(A0[:, p].tolist())
        Q, R = mpmath.qr(Ap, mode="full")
        Rr = R[0:r, 0:n]
        c = (Q.T * mpmath.matrix(b.tolist()))[0:r, 0]
        u = Rr.T * mpmath.lu_solve(Rr * Rr.T, c)
        x = np.zeros(n)
        for i in range(n):
            x[p[i]] = float(u[i])
        return x


@pytest.mark.parametrize("m,n,r,seed", [(12, 6, 3, 0), (9, 5, 5, 1), (15, 8, 1, 2), (20, 10, 7, 3), (10, 10, 4, 4)])
def test_ext_twin_matches_mpmath(coracle, m, n, r, seed):
    rng = np.random.default_rng([m, n, r, seed])
    A0 = np.asfortranarray(rng.standard_normal((m, n)))
    b = rng.standard_normal(m)
    H, alpha, p = M.qrcp_model(A0)[:3]
    x_mp = _mp_cod(A0, p, r, b)
    x_ext = CM.cod_ext(A0, p, r, b)
    assert _rel(x_ext, x_mp) <= 1e-17
    x64 = CM.cod_fp64(coracle, A0, b, r, (H, alpha, p))[0]
    assert _rel(x64, x_mp) <= 1e-13


def test_rank_zero_and_full(coracle):
    A0 = CM.low_rank(120, 30, 30)
    b = np.random.default_rng(5).standard_normal(120)
    fac = M.qrcp_model(A0)[:3]
    assert not CM.cod_fp64(coracle, A0, b, 0, fac)[0].any() and not CM.cod_ext(A0, fac[2], 0, b).any()
    x = CM.cod_fp64(coracle, A0, b, 30, fac)[0]
    assert _rel(x, np.linalg.lstsq(A0, b, rcond=None)[0]) <= 1e-12
