"""Test-side references for the ComplexF64 pivoted factorisation (dhqr_qrcp_c64), next to the tests that use them.

``qrcp_c_model`` restates the device algorithm in numpy, step for step: panels of NB = 32 complex columns in the deferred form
A - V F^H (LAPACK zlaqps), the pivot rule of qrcp_model (largest partial norm, a tie to the smallest index, NaN above every number),
the zlaqps downdate with |r_jc| and tol3z = sqrt(eps), a column that fails it renormed exactly in its deferred state before the next
pivot is chosen, and v = 0, alpha = 0 once the largest remaining norm is exactly 0.  The reflector is that of the library's complex
path (k_house1_c): alpha = -exp(i angle(x0)) ||x||, v = (x - alpha e_0) / sqrt(||x|| (||x|| + |x0|)), so |v|^2 = 2 and
H = I - v v^H; angle sees the signs of a zero x0 (angle(-0 +- 0i) = +-pi, with sin(pi) as numpy has it).  Output in the library's
storage format: v in the lower trapezoid including the diagonal, R above it, diag(R) in alpha, A[:, jpvt] = Q R.

``zgeqp3_refformat`` is LAPACK's complex pivoted QR (scipy.linalg.lapack.zgeqp3): its R, with a real diagonal, and its 0-based
permutation.
"""
from __future__ import annotations

import math

import numpy as np

NB = 32
EPS = np.finfo(np.float64).eps
TOL3Z = np.sqrt(EPS)


def house_c(x):
    """(alpha, v) of the library's complex reflector for a non-zero column x (k_house1_c's formulas, signed-zero pivots included)."""
    s = math.sqrt(float(np.sum(x.real * x.real + x.imag * x.imag)))
    x0 = complex(x[0])
    a0 = math.hypot(x0.real, x0.imag)
    if a0 > 0.0:
        u = complex(x0.real / a0, x0.imag / a0)
    elif math.copysign(1.0, x0.real) > 0:
        u = complex(1.0, x0.imag)
    else:
        u = complex(-1.0, math.copysign(np.sin(np.pi), x0.imag))
    al = complex(-u.real * s, -u.imag * s)
    v = x.copy()
    v[0] = v[0] - al
    return al, v * (1.0 / math.sqrt(s * (s + a0)))


def qrcp_c_model(A0):
    """(H, alpha, jpvt, renorms) of the blocked complex pivoted factorisation of A0 (m x n, n <= m)."""
    A = np.array(A0, dtype=np.complex128, order="F", copy=True)
    m, n = A.shape
    with np.errstate(all="ignore"):
        vn1 = np.sqrt((A.real ** 2 + A.imag ** 2).sum(0))
    vn2 = vn1.copy()
    jpvt = np.arange(n)
    alpha = np.zeros(n, dtype=np.complex128)
    F = np.zeros((n, NB), dtype=np.complex128)
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
                x = A[j:, j] - A[j:, k0:j] @ F[j, :jj].conj()
                nrm = np.sqrt(np.sum(np.abs(x) ** 2))
                if vn1[j] == 0.0 or nrm == 0.0:
                    al, v = 0j, np.zeros_like(x)
                else:
                    al, v = house_c(x)
                A[j:, j] = v
                alpha[j] = al
                if j + 1 >= n:
                    continue
                g = A[j:, k0:j].conj().T @ v                          # V_l^H v
                F[j + 1:, jj] = A[j:, j + 1:].conj().T @ v - F[j + 1:, :jj] @ g
                A[j, j + 1:] -= A[j, k0:j + 1] @ F[j + 1:, :jj + 1].conj().T
                c = np.arange(j + 1, n)
                nz = vn1[c] != 0.0
                t = np.abs(A[j, c]) / np.where(nz, vn1[c], 1.0)
                t = np.maximum(0.0, (1.0 + t) * (1.0 - t))
                t2 = t * (vn1[c] / vn2[c]) ** 2
                flag = nz & (t2 <= TOL3Z)
                upd = nz & ~flag
                vn1[c[upd]] *= np.sqrt(t[upd])
                for cc in c[flag]:
                    r = A[j + 1:, cc] - A[j + 1:, k0:j + 1] @ F[cc, :jj + 1].conj()
                    vn1[cc] = vn2[cc] = np.sqrt(np.sum(np.abs(r) ** 2))
                    renorms += 1
            c1 = k0 + kb
            if c1 < n:
                A[c1:, c1:] -= A[c1:, k0:c1] @ F[c1:, :kb].conj().T
    return A, alpha, jpvt, renorms


def zgeqp3_refformat(a):
    """LAPACK zgeqp3 -> (R, jpvt): R = triu of its n x n block (real diagonal), jpvt 0-based."""
    from scipy.linalg import lapack
    a = np.asfortranarray(a, dtype=np.complex128)
    qr, jpvt, tau, _, info = lapack.zgeqp3(a)
    assert info == 0
    n = a.shape[1]
    return np.triu(qr[:n]), np.asarray(jpvt, dtype=np.int64) - 1


def form_r(H, alpha):
    n = H.shape[1]
    return np.triu(H[:n], 1) + np.diag(alpha)


def form_q(H):
    """Q = H_1 ... H_n [I; 0] from the stored reflectors (H_j = I - v_j v_j^H)."""
    m, n = H.shape
    Q = np.eye(m, n, dtype=np.complex128)
    for j in range(n - 1, -1, -1):
        v = H[j:, j]
        Q[j:] -= np.outer(v, v.conj() @ Q[j:])
    return Q


def nearly_parallel(m, n, seed=0):
    """Complex columns a + 1e-10 g_j: after the first reflector every partial norm collapses by 1e-10, so the downdates fail tol3z."""
    rng = np.random.default_rng([m, n, seed, 17])
    a = rng.standard_normal((m, 1)) + 1j * rng.standard_normal((m, 1))
    return np.asfortranarray(a + 1e-10 * (rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n))))


def low_rank(m, n, r, noise=0.0, seed=3):
    """An m x n complex matrix of exact rank r (singular values 1 .. 1e-3), plus optional complex N(0, noise^2) entries."""
    rng = np.random.default_rng([m, n, r, seed, 1])

    def orth(k, c):
        g = rng.standard_normal((k, c)) + 1j * rng.standard_normal((k, c))
        return np.linalg.qr(g)[0]
    a = (orth(m, r) * np.logspace(0, -3, r)) @ orth(n, r).conj().T
    if noise:
        a = a + noise * (rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n)))
    return np.asfortranarray(a)
