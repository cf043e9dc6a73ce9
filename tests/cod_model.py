"""Test-side references for the complete orthogonal decomposition on the pivoted QR (dhqr_cod_f64, dhqr_solve_cod_f64; DESIGN
§2.8), next to the tests that use them.

At rank r, with A P = Q R: R_r = R[0:r, :] (r x n), R_r' = Z [U; 0], and the minimum-norm solution of the rank-r problem is
x = P Z [U^{-T} (Q'b)[0:r]; 0].

``cod_fp64``: the fp64 twin, stage by stage as the device runs it: a pivoted factorisation in the library's storage format
(``qrcp_model``'s unless one is given), the fp64 oracle's QR of R_r', (Q'b)[0:r] over the first r reflectors, then
``adjoint_oracle.np_solve_adj`` (U^{-T} and Z) and the permutation.
``cod_ext``: the whole solve in long double with no rounding between the stages (tests/cod_ext.c, compiled on first use into a
temporary directory, like adjoint_oracle's adj_ext), for a given permutation and rank.
``pinv_solve``: the minimum-norm solution of the rank-r truncation by SVD, the answer numpy.linalg.lstsq gives on an exactly
rank-r matrix.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import adjoint_oracle as AO
import matrix_families as F
import qrcp_model as M


def rr_t(H, alpha, r):
    """R_r' (n x r, Fortran order) from a factorisation in the library's storage format."""
    return np.asfortranarray(M.form_r(H, alpha)[:r].T)


def cod_fp64(coracle, A0, b, r, fac=None):
    """(x, F, gamma): the fp64 twin of dhqr_cod_f64 + dhqr_solve_cod_f64 at rank r.  ``fac`` = (H, alpha, jpvt) of A0, default
    qrcp_model's.  ``b``: length m, or (m, k)."""
    H, alpha, jpvt = fac if fac is not None else M.qrcp_model(A0)[:3]
    m, n = A0.shape
    b2 = np.reshape(np.asarray(b, dtype=np.float64), (m, -1))
    x = np.zeros((n, b2.shape[1]))
    F = gamma = None
    if r > 0:
        F, gamma = coracle.qr(rr_t(H, alpha, r))
        Hr = np.asfortranarray(H[:, :r])
        for k in range(b2.shape[1]):
            c = coracle.apply_qt(Hr, b2[:, k].copy())[:r]
            x[jpvt, k] = AO.np_solve_adj(F, gamma, c)
    return (x[:, 0] if np.ndim(b) == 1 else x), F, gamma


_HERE = os.path.dirname(os.path.abspath(__file__))
_clib = None


def _lib():
    global _clib
    if _clib is None:
        out = tempfile.mkdtemp(prefix="cod_ext_")
        so = os.path.join(out, "libcod_ext.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-fopenmp", "-std=c11", "-shared", "-o", so, os.path.join(_HERE, "cod_ext.c"), "-lm"])
        lib = C.CDLL(so)
        shutil.rmtree(out, ignore_errors=True)          # the mapping outlives the file: nothing is left behind
        i64, vp, ci = C.c_int64, C.c_void_p, C.c_int
        lib.cod_ext.argtypes = [i64, i64, i64, vp, i64, ci, vp, i64, vp, ci]
        lib.cod_ext.restype = ci
        _clib = lib
    return _clib


def cod_ext(A0, jpvt, r, b):
    """x = P Z [U^{-T} (Q'b)[0:r]; 0] in long double, rounded to double, for the permutation ``jpvt`` (0-based, the device's or
    a model's) and rank ``r``.  ``b``: length m, or (m, k)."""
    ap = np.asfortranarray(np.asarray(A0, dtype=np.float64)[:, jpvt])
    m, n = ap.shape
    b2 = np.asfortranarray(np.reshape(np.asarray(b, dtype=np.float64), (m, -1)))
    k = b2.shape[1]
    u = np.zeros((n, k), order="F")
    p = lambda t: None if t.size == 0 else C.c_void_p(t.ctypes.data)
    rc = _lib().cod_ext(m, n, int(r), p(ap), max(m, 1), k, p(b2), max(m, 1), p(u), os.cpu_count() or 1)
    if rc:
        raise RuntimeError(f"cod_ext rc={rc}")
    x = np.zeros((n, k))
    x[jpvt] = u
    return x[:, 0] if np.ndim(b) == 1 else x


def pinv_solve(A0, b, r):
    """The minimum-norm least-squares solution of the rank-r truncation of A0 (SVD)."""
    u, s, vt = np.linalg.svd(A0, full_matrices=False)
    return vt[:r].T @ ((u[:, :r].T @ b) / (s[:r] if np.ndim(b) == 1 else s[:r, None]))


def low_rank(m, n, r, noise=0.0, seed=3):
    """A rank-r m x n matrix with singular values logspace(0, -3, r) (kappa_r = 1e3), plus optional Gaussian noise; the inputs
    of test_gpu_qrcp.py's rank tests."""
    rng = np.random.default_rng([m, n, r, seed])
    a = (F._orth(rng, m, r) * np.logspace(0, -3, r)) @ F._orth(rng, n, r).T
    if noise:
        a = a + noise * rng.standard_normal((m, n))
    return np.asfortranarray(a)
