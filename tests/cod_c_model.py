"""Test-side reference for the ComplexF64 complete orthogonal decomposition solve (dhqr_solve_cod_c64), next to the tests that use it.

``cod_ext_c``: the whole solve, x = P Z [U^{-H} (Q^H b)[0:r]; 0], in long double with no rounding between the stages, for a given
permutation and rank (tests/cod_ext_c.c, compiled on first use into a temporary directory, as cod_model does for cod_ext.c).
``pinv_solve_c``: the minimum-norm least-squares solution of the rank-r truncation (SVD).
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_clib = None


def _lib():
    global _clib
    if _clib is None:
        out = tempfile.mkdtemp(prefix="cod_ext_c_")
        so = os.path.join(out, "libcod_ext_c.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-fopenmp", "-std=c11", "-shared", "-o", so, os.path.join(_HERE, "cod_ext_c.c"), "-lm"])
        lib = C.CDLL(so)
        shutil.rmtree(out, ignore_errors=True)          # the mapping outlives the file: nothing is left behind
        i64, vp, ci = C.c_int64, C.c_void_p, C.c_int
        lib.cod_ext_c.argtypes = [i64, i64, i64, vp, i64, ci, vp, i64, vp, ci]
        lib.cod_ext_c.restype = ci
        _clib = lib
    return _clib


def cod_ext_c(A0, jpvt, r, b):
    """x = P Z [U^{-H} (Q^H b)[0:r]; 0] in long double, rounded to ComplexF64, for the permutation ``jpvt`` (0-based) and rank ``r``.
    ``b``: length m, or (m, k)."""
    ap = np.asfortranarray(np.asarray(A0, dtype=np.complex128)[:, jpvt])
    m, n = ap.shape
    b2 = np.asfortranarray(np.reshape(np.asarray(b, dtype=np.complex128), (m, -1)))
    k = b2.shape[1]
    u = np.zeros((n, k), dtype=np.complex128, order="F")
    p = lambda t: None if t.size == 0 else C.c_void_p(t.ctypes.data)
    rc = _lib().cod_ext_c(m, n, int(r), p(ap), max(m, 1), k, p(b2), max(m, 1), p(u), os.cpu_count() or 1)
    if rc:
        raise RuntimeError(f"cod_ext_c rc={rc}")
    x = np.zeros((n, k), dtype=np.complex128)
    x[jpvt] = u
    return x[:, 0] if np.ndim(b) == 1 else x


def pinv_solve_c(A0, b, r):
    """The minimum-norm least-squares solution of the rank-r truncation of complex A0 (SVD)."""
    u, s, vh = np.linalg.svd(A0, full_matrices=False)
    return vh[:r].conj().T @ ((u[:, :r].conj().T @ b) / (s[:r] if np.ndim(b) == 1 else s[:r, None]))
