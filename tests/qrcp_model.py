"""Test-side references for the pivoted factorisation (dhqr_qrcp_f64), next to the tests that use them.

``qrcp_model`` restates the device algorithm in numpy, step for step: panels of NB = 32 columns in the deferred form A - V F'
(LAPACK dlaqps), the pivot rule (largest partial norm, a tie to the smallest index, NaN above every number: numpy argmax), the
dlaqps downdate with tol3z = sqrt(eps), a column that fails it renormed exactly in its deferred state before the next pivot is
chosen, and v = 0, alpha = 0 once the largest remaining norm is exactly 0.  Output in the library's storage format: v scaled to
|v|^2 = 2 in the lower trapezoid including the diagonal, R above it, diag(R) in alpha, A[:, jpvt] = Q R.

``dgeqp3_refformat`` is LAPACK's pivoted QR (scipy.linalg.lapack.dgeqp3) converted to the same format, as
oracle.lapack_qr_refformat does for dgeqrf.
"""
from __future__ import annotations

import numpy as np

NB = 32
EPS = np.finfo(np.float64).eps
TOL3Z = np.sqrt(EPS)


def qrcp_model(A0):
    """(H, alpha, jpvt, renorms) of the blocked pivoted factorisation of A0 (m x n, n <= m)."""
    A = np.array(A0, dtype=np.float64, order="F", copy=True)
    m, n = A.shape
    with np.errstate(all="ignore"):
        vn1 = np.sqrt((A * A).sum(0))
    vn2 = vn1.copy()
    jpvt = np.arange(n)
    alpha = np.zeros(n)
    F = np.zeros((n, NB))
    renorms = 0
    with np.errstate(all="ignore"):
        for k0 in range(0, n, NB):
            kb = min(NB, n - k0)
            for jj in range(kb):
                j = k0 + jj
                p = j + int(np.argmax(vn1[j:]))
                if p != j:
                    A[:, [j, p]] = A[:, [p, j]]
                    vn1[[j, p]] = vn1[[p, j]]
                    vn2[[j, p]] = vn2[[p, j]]
                    jpvt[[j, p]] = jpvt[[p, j]]
                    F[[j, p], :jj] = F[[p, j], :jj]
                x = A[j:, j] - A[j:, k0:j] @ F[j, :jj]
                nrm = np.sqrt(x @ x)
                if vn1[j] == 0.0 or nrm == 0.0:
                    al, v = 0.0, np.zeros_like(x)
                else:
                    al = -nrm if x[0] >= 0.0 else nrm
                    v = x.copy()
                    v[0] -= al
                    v *= 1.0 / np.sqrt(nrm * (nrm + abs(x[0])))
                A[j:, j] = v
                alpha[j] = al
                if j + 1 >= n:
                    continue
                g = A[j:, k0:j].T @ v
                F[j + 1:, jj] = A[j:, j + 1:].T @ v - F[j + 1:, :jj] @ g
                A[j, j + 1:] -= F[j + 1:, :jj + 1] @ A[j, k0:j + 1]
                c = np.arange(j + 1, n)
                nz = vn1[c] != 0.0
                t = np.abs(A[j, c]) / np.where(nz, vn1[c], 1.0)
                t = np.maximum(0.0, (1.0 + t) * (1.0 - t))
                t2 = t * (vn1[c] / vn2[c]) ** 2
                flag = nz & (t2 <= TOL3Z)
                upd = nz & ~flag
                vn1[c[upd]] *= np.sqrt(t[upd])
                for cc in c[flag]:
                    r = A[j + 1:, cc] - A[j + 1:, k0:j + 1] @ F[cc, :jj + 1]
                    vn1[cc] = vn2[cc] = np.sqrt(r @ r)
                    renorms += 1
            c1 = k0 + kb
            if c1 < n:
                A[c1:, c1:] -= A[c1:, k0:c1] @ F[c1:, :kb].T
    return A, alpha, jpvt, renorms


def dgeqp3_refformat(a):
    """LAPACK dgeqp3 -> (H, alpha, jpvt) in the library's format; jpvt 0-based."""
    from scipy.linalg import lapack
    a = np.asfortranarray(a, dtype=np.float64)
    qr, jpvt, tau, _, info = lapack.dgeqp3(a)
    assert info == 0
    n = a.shape[1]
    h = np.asfortranarray(qr.copy())
    alpha = np.diag(qr)[:n].copy()
    for j in range(n):
        st = -np.sign(alpha[j]) * np.sqrt(tau[j])
        h[j + 1:, j] = qr[j + 1:, j] * st
        h[j, j] = st
    return h, alpha, np.asarray(jpvt, dtype=np.int64) - 1


def form_r(H, alpha):
    n = H.shape[1]
    return np.triu(H[:n], 1) + np.diag(alpha)


def pivot_gap(R):
    """Smallest relative gap between the chosen norm |R[k, k]| and the runner-up max_{c > k} ||R[k:c+1, c]|| over the steps."""
    n = R.shape[1]
    tail = np.sqrt(np.cumsum((R * R)[::-1], axis=0)[::-1])      # tail[k, c] = ||R[k:, c]||
    gaps = [(abs(R[k, k]) - tail[k, k + 1:].max()) / abs(R[k, k]) for k in range(n - 1)]
    return float(min(gaps))


def nearly_parallel(m, n, seed=0):
    """Columns a + 1e-10 g_j: after the first reflector every partial norm collapses by 1e-10, so the downdates fail tol3z."""
    rng = np.random.default_rng([m, n, seed, 7])
    a = rng.standard_normal((m, 1))
    return np.asfortranarray(a + 1e-10 * rng.standard_normal((m, n)))
