"""CPU check of tests/append_model.py, the blocked restatement of dhqr_qr_append_f64 / dhqr_apply_qt_append_f64 (DESIGN §2.10),
against LAPACK's triangular-pentagonal QR (scipy dtpqrt / dtpmqrt) and against the oracle's factorisation of the stacked
matrix [R; B], whose reflectors restricted to their nonzero rows are (vtop, V2)."""
import numpy as np
import pytest
from scipy.linalg import lapack

import append_model as M
import matrix_families as F

SHAPES = [(1, 1), (1, 5), (31, 2), (33, 33), (128, 31), (129, 255), (200, 64), (260, 600)]


def start(n, seed):
    """R of an existing factorisation (the oracle's qr of a random tall matrix) and its alpha."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n + 7, n))
    Q, R = np.linalg.qr(A)
    return np.triu(R, 1) + np.tril(rng.standard_normal((n, n))), np.diag(R).copy()   # junk below the diagonal is never read


@pytest.mark.parametrize("n,k", SHAPES)
def test_against_dtpqrt(n, k):
    Rj, alpha = start(n, n + k)
    B = np.random.default_rng(k).standard_normal((k, n))
    R1, a1, V2, vtop = M.qr_append(Rj, alpha, B)
    assert np.array_equal(np.tril(R1), np.tril(Rj)), "the diagonal and lower part of R were written"
    Rfull = np.triu(Rj, 1) + np.diag(alpha)
    nb = min(n, 32)
    a, b, t, info = lapack.dtpqrt(0, nb, np.asfortranarray(Rfull), np.asfortranarray(B))
    assert info == 0
    scale = np.linalg.norm(np.vstack([Rfull, B]), axis=0)
    assert np.abs(np.triu(R1, 1) - np.triu(a, 1)).max(initial=0) <= 1e-13 * scale.max()
    assert np.abs(a1 - np.diag(a)).max() <= 1e-13 * scale.max()
    tau, v = M.lapack_form(V2, vtop)
    assert np.allclose(tau, t[np.arange(n) % nb, np.arange(n)], rtol=1e-12, atol=1e-14)
    assert np.allclose(v, b, rtol=1e-11, atol=1e-12)
    assert np.allclose((V2 ** 2).sum(0) + vtop ** 2, 2.0, atol=1e-13)
    # the apply functions against dtpmqrt on the same reflectors
    c = np.random.default_rng(3).standard_normal((n, 3))
    e = np.random.default_rng(4).standard_normal((k, 3))
    cq, eq = M.apply_append(V2, vtop, c, e)
    cl, el, info = lapack.dtpmqrt(0, np.asfortranarray(b), np.asfortranarray(t), np.asfortranarray(c), np.asfortranarray(e),
                                  trans="T")
    assert info == 0
    assert np.allclose(cq, cl, atol=1e-12) and np.allclose(eq, el, atol=1e-12)
    cb, eb = M.apply_append(V2, vtop, cq, eq, trans=True)
    assert np.allclose(cb, c, atol=1e-12) and np.allclose(eb, e, atol=1e-12)


@pytest.mark.parametrize("family", ["uniform", "normal", "colscale", "rowscale"])
@pytest.mark.parametrize("n,k", [(40, 17), (130, 300), (257, 64)])
def test_against_stacked_oracle(coracle, family, n, k):
    """R from the oracle's factorisation of a family matrix, B from the same family: the oracle on [R; B] has R' above its diagonal,
    vtop on it, zeros below it in the R block and V2 below row n."""
    A = F.make(family, n + k + n, n)
    H0, a0 = coracle.qr(np.asfortranarray(A[:n + 5]))
    R = np.triu(H0[:n], 1)
    B = np.asfortranarray(A[n + 5:n + 5 + k])
    S = np.asfortranarray(np.vstack([R + np.diag(a0), B]))
    Hs, as_ = coracle.qr(S.copy(order="F"))              # the oracle factors in place
    R1, a1, V2, vtop = M.qr_append(R, a0, B)
    scale = np.linalg.norm(S, axis=0)
    tol = 64 * np.linalg.cond(S / scale) * np.finfo(float).eps     # both are backward stable: forward errors scale with kappa
    assert (np.abs(np.triu(R1 - Hs[:n], 1)) / scale).max(initial=0) <= tol
    assert (np.abs(a1 - as_) / scale).max() <= tol
    assert np.abs(vtop - np.diag(Hs[:n])).max() <= tol
    assert np.abs(np.tril(Hs[:n], -1)).max(initial=0) == 0.0
    assert np.abs(V2 - Hs[n:]).max() <= tol


def test_from_zero():
    """Starting from R = 0, alpha = 0 (a zero x0 counts as positive, unlike the reference's sign(0) = 0): R'R' = B'B and the
    least-squares solution of a block fed in pieces equals lstsq of the whole."""
    rng = np.random.default_rng(0)
    n, blocks = 45, [1, 30, 77, 3, 60]
    A = rng.standard_normal((sum(blocks), n))
    b = rng.standard_normal(sum(blocks))
    R, alpha, c, ss, r0 = np.zeros((n, n)), np.zeros(n), np.zeros((n, 1)), 0.0, 0
    for kb in blocks:
        R, alpha, V2, vtop = M.qr_append(R, alpha, A[r0:r0 + kb])
        c, e = M.apply_append(V2, vtop, c, b[r0:r0 + kb, None])
        ss += float((e ** 2).sum())
        r0 += kb
    Rf = np.triu(R, 1) + np.diag(alpha)
    assert np.allclose(Rf.T @ Rf, A.T @ A, atol=1e-10 * np.abs(A.T @ A).max())
    x = np.linalg.solve(Rf, c[:, 0])
    xl, res, *_ = np.linalg.lstsq(A, b, rcond=None)
    assert np.allclose(x, xl, atol=1e-11)
    assert np.isclose(ss, float(res[0]), rtol=1e-10)
