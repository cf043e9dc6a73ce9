"""References for the solves with the adjoint (test infrastructure only).

``adj_ext(a, c)``: z = R^{-H} c and y = Q [z; 0], the minimum-norm solution of A^H y = c, with the factorisation and both
solves in long double (tests/adjoint_ext.c, compiled on first use into a temporary directory, like test_abi.py's C consumer).
``np_forwardsolve`` / ``np_solve_adj`` and their complex twins: the same in fp64 on a given factorisation (H, alpha) in the
library's storage format, following the reference's row-oriented recurrence mirrored: z_i = (c_i - sum_{j<i} conj(H[j,i]) z_j)
/ conj(alpha_i).
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def _load():
    global _lib
    if _lib is None:
        out = tempfile.mkdtemp(prefix="adjoint_ext_")
        so = os.path.join(out, "libadjoint_ext.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-fopenmp", "-std=c11", "-shared", "-o", so, os.path.join(_HERE, "adjoint_ext.c"), "-lm"])
        lib = C.CDLL(so)
        shutil.rmtree(out, ignore_errors=True)          # the mapping outlives the file: nothing is left behind
        i64, vp, ci = C.c_int64, C.c_void_p, C.c_int
        lib.adj_ext.argtypes = [i64, i64, vp, i64, ci, ci, vp, i64, vp, vp, ci]
        lib.adj_ext.restype = ci
        _lib = lib
    return _lib


def adj_ext(a, c):
    """(z, y) in long double, rounded to double, shaped like ``c`` (y with m rows); ``a`` is the input matrix (m x n), ``c``
    length n or n x k.  Float64 or ComplexF64 after the dtypes of ``a`` and ``c``."""
    cplx = np.iscomplexobj(a) or np.iscomplexobj(c)
    dt = np.complex128 if cplx else np.float64
    a = np.asfortranarray(a, dtype=dt)
    m, n = a.shape
    cc = np.asarray(c, dtype=dt)
    cc = np.asfortranarray(cc.reshape(n, cc.shape[1] if cc.ndim == 2 else 1))
    k = cc.shape[1]
    z = np.zeros((n, k), dtype=dt, order="F")
    y = np.zeros((m, k), dtype=dt, order="F")
    p = lambda t: None if t.size == 0 else C.c_void_p(t.ctypes.data)
    rc = _load().adj_ext(m, n, p(a), max(m, 1), int(cplx), k, p(cc), max(n, 1), p(z), p(y), os.cpu_count() or 1)
    if rc:
        raise RuntimeError(f"adj_ext rc={rc}")
    if np.ndim(c) == 1:
        return z[:, 0], y[:, 0]
    return z, y


def np_forwardsolve(h, alpha, c):
    """z = R^{-T} c with R = triu(h, 1) + diag(alpha), row by row: z_i = (c_i - sum_{j<i} h[j, i] z_j) / alpha_i."""
    n = h.shape[1]
    z = np.array(c, dtype=np.float64, copy=True)[:n]
    for i in range(n):
        z[i] = (z[i] - h[:i, i] @ z[:i]) / alpha[i]
    return z


def np_solve_adj(h, alpha, c):
    """The minimum-norm solution of A^T y = c: y = Q [R^{-T} c; 0], Q = H_1 ... H_n (the reflectors in reverse order)."""
    m, n = h.shape
    y = np.zeros((m,) + np.shape(c)[1:])
    y[:n] = np_forwardsolve(h, alpha, c)
    for j in range(n - 1, -1, -1):
        y[j:] -= np.multiply.outer(h[j:, j], h[j:, j] @ y[j:])
    return y


def np_forwardsolve_c(h, alpha, c):
    """z = R^{-H} c: z_i = (c_i - sum_{j<i} conj(h[j, i]) z_j) / conj(alpha_i)."""
    n = h.shape[1]
    z = np.array(c, dtype=np.complex128, copy=True)[:n]
    for i in range(n):
        z[i] = (z[i] - np.conj(h[:i, i]) @ z[:i]) / np.conj(alpha[i])
    return z


def np_solve_adj_c(h, alpha, c):
    """The minimum-norm solution of A^H y = c: y = Q [R^{-H} c; 0] with H_j = I - v_j v_j^H."""
    m, n = h.shape
    y = np.zeros((m,) + np.shape(c)[1:], dtype=np.complex128)
    y[:n] = np_forwardsolve_c(h, alpha, c)
    for j in range(n - 1, -1, -1):
        y[j:] -= np.multiply.outer(h[j:, j], np.conj(h[j:, j]) @ y[j:])
    return y
