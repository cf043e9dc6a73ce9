"""CPU check of tests/downdate_model.py, the blocked restatement of dhqr_qr_downdate_f64 / dhqr_apply_downdate_f64 (DESIGN §2.11):
against the unblocked recurrence (in fp64 and in long double, tests/downdate_ext.c), against numpy's QR of the remaining rows up to
row signs, against the Gram identity R''R' = R'R - Z'Z and least squares on the remaining rows, through append / downdate round
trips, and on the failure rule."""
import numpy as np
import pytest

import append_model as AM
import downdate_model as M

SHAPES = [(1, 1), (5, 1), (31, 2), (33, 33), (64, 31), (129, 40), (200, 64), (260, 100)]


def factor(A):
    """(R in the library's storage with junk below the diagonal, alpha) of A."""
    R = np.linalg.qr(A, mode="r")
    n = R.shape[1]
    return np.triu(R, 1) + np.tril(np.full((n, n), 7.0)), np.diag(R).copy()


def full(R, alpha):
    return np.triu(R, 1) + np.diag(alpha)


def signed(R):
    """Rows scaled to a positive diagonal: R up to row signs."""
    d = np.sign(np.diag(R))
    d[d == 0] = 1.0
    return d[:, None] * R


def problem(n, k, seed, extra=60):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((k + n + extra, n))
    b = rng.standard_normal((A.shape[0], 2))
    return A, b


@pytest.mark.parametrize("n,k", SHAPES)
def test_blocked_matches_unblocked_and_remaining_rows(n, k):
    A, _ = problem(n, k, n * 7 + k)
    R, alpha = factor(A)
    R1, a1, V2, vt, info = M.qr_downdate(R, alpha, A[:k])
    assert info == 0
    assert np.array_equal(np.tril(R1), np.tril(R)), "the diagonal and lower part of R were written"
    Ru, au, V2u, vtu, infou = M.unblocked(R, alpha, A[:k])
    Re, ae, V2e, vte, infoe = M.ext_downdate(R, alpha, A[:k])
    assert infou == infoe == 0
    scale = np.linalg.norm(A, 2)
    for got in ((full(R1, a1), V2, vt), (full(Ru, au), V2u, vtu)):
        assert np.abs(got[0] - full(Re, ae)).max() <= 1e-12 * scale
        assert np.abs(got[1] - V2e).max() <= 1e-11 and np.abs(got[2] - vte).max() <= 1e-11
    # the hyperbolic norm of every reflector is 2
    assert np.allclose(vt ** 2 - (V2 ** 2).sum(0), 2.0, atol=1e-10)
    # R' is the R of the remaining rows, up to row signs, and obeys the Gram identity
    Rrem = np.linalg.qr(A[k:], mode="r")
    assert np.abs(signed(full(R1, a1)) - signed(Rrem)).max() <= 1e-12 * scale
    G = full(R, alpha).T @ full(R, alpha) - A[:k].T @ A[:k]
    assert np.abs(full(R1, a1).T @ full(R1, a1) - G).max() <= 1e-12 * scale ** 2


@pytest.mark.parametrize("n,k", [(33, 33), (129, 40), (200, 64)])
def test_least_squares_and_residual(n, k):
    A, b = problem(n, k, 3 * n + k)
    Q, Rr = np.linalg.qr(A)
    R, alpha = factor(A)
    R, alpha = np.triu(Rr, 1) + np.tril(R, -1), np.diag(Rr).copy()     # the same Q and R, so c = Q'b matches
    c = Q.T @ b
    rss = ((b - A @ np.linalg.lstsq(A, b, rcond=None)[0]) ** 2).sum(0)
    R1, a1, V2, vt, info = M.qr_downdate(R, alpha, A[:k])
    c1, e1 = M.apply_downdate(V2, vt, c, b[:k])
    x = np.linalg.solve(full(R1, a1), c1)
    xr, res = np.linalg.lstsq(A[k:], b[k:], rcond=None)[:2]
    assert np.abs(x - xr).max() <= 1e-12 * np.abs(xr).max()
    assert np.allclose(rss - (e1 ** 2).sum(0), res, rtol=1e-11)
    Ru, au, V2u, vtu, _, cu, eu = M.unblocked(R, alpha, A[:k], c, b[:k])
    ce, ee = M.ext_downdate(R, alpha, A[:k], c, b[:k])[5:]
    assert np.abs(c1 - ce).max() <= 1e-12 * np.abs(ce).max() and np.abs(e1 - ee).max() <= 1e-12 * np.abs(ee).max()
    assert np.abs(cu - ce).max() <= 1e-12 * np.abs(ce).max()


@pytest.mark.parametrize("n,k", [(40, 17), (150, 64)])
def test_append_and_downdate_round_trips(n, k):
    A, _ = problem(n, k, n + 11 * k)
    R, alpha = factor(A[k:])
    Ra, aa = AM.qr_append(R, alpha, A[:k])[:2]                        # append then downdate the same rows
    Rd, ad, _, _, info = M.qr_downdate(Ra, aa, A[:k])
    assert info == 0
    assert np.abs(signed(full(Rd, ad)) - signed(full(R, alpha))).max() <= 1e-11 * np.linalg.norm(A, 2)
    R, alpha = factor(A)                                              # downdate then append
    Rd, ad = M.qr_downdate(R, alpha, A[:k])[:2]
    Ra, aa = AM.qr_append(Rd, ad, A[:k])[:2]
    assert np.abs(signed(full(Ra, aa)) - signed(full(R, alpha))).max() <= 1e-11 * np.linalg.norm(A, 2)


@pytest.mark.parametrize("n,bad", [(64, 0), (64, 20), (200, 37), (300, 170)])
def test_failure_rule(n, bad):
    """Real rows plus a row that was never added, zero before column `bad` and large at it: the downdate fails exactly there, in
    the first panel or a later one; from that column on vtop = 0, V2 = 0, alpha = NaN, and the rows above it are the exact
    downdate of the real rows."""
    k = 9
    A, _ = problem(n, k, n + bad)
    R, alpha = factor(A)
    Z = A[:k + 1].copy()
    Z[k] = 0.0
    Z[k, bad:] = 100.0 * np.linalg.norm(A, 2)
    R1, a1, V2, vt, info = M.qr_downdate(R, alpha, Z)
    assert info == bad + 1
    assert np.isnan(a1[bad:]).all() and not np.isnan(a1[:bad]).any()
    assert (vt[bad:] == 0).all() and (V2[:, bad:] == 0).all()
    Rrem = np.linalg.qr(A[k:], mode="r")
    top = full(R1, np.nan_to_num(a1))[:bad]
    assert np.abs(signed(top) - signed(Rrem)[:bad]).max(initial=0) <= 1e-11 * np.linalg.norm(A, 2)
    assert np.array_equal(np.triu(R1, 1)[bad:], np.triu(R, 1)[bad:]), "rows from the failed column on are left as they were"
    assert M.unblocked(R, alpha, Z)[4] == M.ext_downdate(R, alpha, Z)[4] == bad + 1
    # a row that was never added, in full: fails somewhere, and a zero column from a zero column does not fail
    assert M.qr_downdate(R, alpha, 10 * A[:1])[4] > 0
    Rz, az = np.zeros((3, 3)), np.zeros(3)
    assert M.qr_downdate(Rz, az, np.zeros((2, 3)))[4] == 0
