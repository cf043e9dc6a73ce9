"""CPU oracle for DistributedHouseholderQR.jl's hot path — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product path (libdhqr.so + the dhqr_b200 host package) never does.

Four things live here, each citing the reference lines it follows
(S:n = line n of the reference's src/DistributedHouseholderQR.jl, T:n = test/runtests.jl:n):

* ``COracle``  — ctypes binding of oracle/dhqr_oracle.c (the C restatement, OpenMP threads over
  trailing-column chunks like S:203-211), including ``qr_ext`` / ``qr_ext_c``: the same recurrences in long double, the
  yardstick for the accuracy of both the fp64 oracle and the library.
* ``np_*``     — a pure-numpy twin of the same recurrences (small cases; independent code path).
* ``np_*_c``   — the same recurrences for ComplexF64 (S:9, S:51-59, S:162-196; the reference tests both element types,
  T:43): oracle only so far, there is no complex CUDA path to check against it yet.
* ``lapack_*`` — LAPACK dgeqrf mapped into the reference's storage format (alpha = diag R,
  triu(H,1) = triu(R,1), v_ref = -sign(alpha) * sqrt(tau) * [1; v_lapack], SURVEY App. A): the "stdlib" comparator
  the reference's own tests normalise to (T:49-51).

Parity status: no golden vectors exist in the reference and Julia is absent, so bitwise parity with
the Julia binary is UNPINNED; the oracle is pinned by the reference's own test properties
(T:51,62,81; test/partialdot.jl:15-19), by LAPACK, and by tests/golden/ fixtures.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libdhqr_oracle.so")


def build(force: bool = False) -> str:
    """Compile oracle/dhqr_oracle.c with the committed Makefile (gcc + OpenMP)."""
    src = os.path.join(_HERE, "dhqr_oracle.c")
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "libdhqr_oracle.so"])
    return _LIB


class _Block(C.Structure):
    _fields_ = [("a", C.c_void_p), ("lda", C.c_int64), ("col0", C.c_int64), ("ncols", C.c_int64)]


def _fptr(x: np.ndarray) -> C.c_void_p:
    assert x.dtype == np.float64
    return C.c_void_p(x.ctypes.data)


def _check_colmajor(a: np.ndarray):
    assert a.dtype == np.float64 and a.ndim == 2 and a.flags.f_contiguous, "need Fortran-order float64"


class COracle:
    """ctypes face of oracle/dhqr_oracle.c."""

    def __init__(self):
        self.lib = C.CDLL(build())
        L = self.lib
        i64, dbl, vp, ci = C.c_int64, C.c_double, C.c_void_p, C.c_int
        L.dhqr_oracle_alphafactor.restype = dbl
        L.dhqr_oracle_alphafactor.argtypes = [dbl]
        L.dhqr_oracle_partialdot.restype = dbl
        L.dhqr_oracle_partialdot.argtypes = [vp, vp, i64, i64]
        L.dhqr_oracle_qr.argtypes = [i64, i64, vp, i64, vp, ci]
        L.dhqr_oracle_qr_steps.argtypes = [i64, i64, vp, i64, vp, i64, ci, C.POINTER(dbl)]
        L.dhqr_oracle_qr_steps_strided.argtypes = [i64, i64, vp, i64, vp, i64, i64, ci, C.POINTER(dbl)]
        L.dhqr_oracle_householder_blocks.argtypes = [i64, i64, ci, C.POINTER(_Block), vp, ci]
        L.dhqr_oracle_apply_qt_blocks.argtypes = [i64, i64, ci, C.POINTER(_Block), vp]
        L.dhqr_oracle_backsolve_blocks.argtypes = [i64, i64, ci, C.POINTER(_Block), vp, vp]
        L.dhqr_oracle_solve_blocks.argtypes = [i64, i64, ci, C.POINTER(_Block), vp, vp]
        L.dhqr_oracle_apply_qt.argtypes = [i64, i64, vp, i64, vp]
        L.dhqr_oracle_backsolve.argtypes = [i64, i64, vp, i64, vp, vp]
        L.dhqr_oracle_ldiv.argtypes = [i64, i64, vp, i64, vp, vp, vp]
        L.dhqr_oracle_uniform.restype = dbl
        L.dhqr_oracle_uniform.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64]
        L.dhqr_oracle_fill_uniform.restype = None
        L.dhqr_oracle_fill_uniform.argtypes = [C.c_uint64, i64, i64, i64, i64, vp, i64]
        L.dhqr_oracle_max_threads.restype = ci
        L.dhqr_oracle_ext_mant_dig.restype = ci
        L.dhqr_oracle_qr_ext.argtypes = [i64, i64, vp, i64, vp, ci, vp, i64, vp, vp, vp, ci]
        L.dhqr_oracle_qr_ext_c.argtypes = [i64, i64, vp, i64, vp, ci, vp, i64, vp, vp, ci]

    # -- scalars / primitives -------------------------------------------------
    def max_threads(self) -> int:
        return int(self.lib.dhqr_oracle_max_threads())

    def ext_mant_dig(self) -> int:
        """Significand bits of the extended-precision reference (LDBL_MANT_DIG: 64 on x86-64, 113 on aarch64)."""
        return int(self.lib.dhqr_oracle_ext_mant_dig())

    # -- extended-precision reference (same recurrences in long double) ---------------------------------------------
    def _ext(self, a, b, nthreads, want_qb, cplx):
        dt = np.complex128 if cplx else np.float64
        h = np.array(a, dtype=dt, order="F", copy=True)
        m, n = h.shape
        alpha = np.zeros(n, dtype=dt)
        bb = None if b is None else np.asfortranarray(np.asarray(b, dtype=dt).reshape(m, -1))
        k = 0 if bb is None else bb.shape[1]
        qtb = np.zeros((m, k), dtype=dt, order="F")
        qb = np.zeros((m, k), dtype=dt, order="F") if want_qb else None
        x = np.zeros((n, k), dtype=dt, order="F")
        if nthreads <= 0:
            nthreads = self.max_threads()
        p = lambda t: None if t is None or t.size == 0 else C.c_void_p(t.ctypes.data)
        lda, ldb = max(m, 1), max(m, 1)
        if cplx:
            rc = self.lib.dhqr_oracle_qr_ext_c(m, n, p(h), lda, p(alpha), k, p(bb), ldb, p(qtb), p(x), nthreads)
        else:
            rc = self.lib.dhqr_oracle_qr_ext(m, n, p(h), lda, p(alpha), k, p(bb), ldb, p(qtb), p(qb), p(x), nthreads)
        if rc:
            raise RuntimeError(f"dhqr_oracle_qr_ext rc={rc}")
        return h, alpha, qtb, qb, x

    def qr_ext(self, a: np.ndarray, b=None, nthreads: int = 0, want_qb: bool = False):
        """qr!(A) in long double, rounded to double: returns (H, alpha) without touching ``a``.  With ``b`` (length m, or
        m x k) the right-hand sides go through the long double factorisation as well and the result is
        (H, alpha, Q'b, Qb or None, H \\ b), each of shape (m, k) / (n, k)."""
        h, alpha, qtb, qb, x = self._ext(a, b, nthreads, want_qb, False)
        return (h, alpha) if b is None else (h, alpha, qtb, qb, x)

    def apply_qt_ext(self, a: np.ndarray, b: np.ndarray, nthreads: int = 0) -> np.ndarray:
        """Q'b (S:232-242) with Q from the long double factorisation of ``a`` (the input matrix, not H)."""
        return self._ext(a, b, nthreads, False, False)[2].reshape(np.shape(b))

    def ldiv_ext(self, a: np.ndarray, b: np.ndarray, nthreads: int = 0) -> np.ndarray:
        """qr!(A) \\ b (S:317-321) entirely in long double; ``a`` is the input matrix."""
        x = self._ext(a, b, nthreads, False, False)[4]
        return x[:, 0] if np.ndim(b) == 1 else x

    def qr_ext_c(self, a: np.ndarray, b=None, nthreads: int = 0):
        """ComplexF64 twin of qr_ext (np_qr_c / np_apply_qt_c in long double): (H, alpha) or (H, alpha, Q'b, H \\ b)."""
        h, alpha, qtb, _, x = self._ext(a, b, nthreads, False, True)
        return (h, alpha) if b is None else (h, alpha, qtb, x)

    def ldiv_ext_c(self, a: np.ndarray, b: np.ndarray, nthreads: int = 0) -> np.ndarray:
        x = self._ext(a, b, nthreads, False, True)[4]
        return x[:, 0] if np.ndim(b) == 1 else x

    def alphafactor(self, x: float) -> float:
        return float(self.lib.dhqr_oracle_alphafactor(float(x)))

    def partialdot(self, a: np.ndarray, b: np.ndarray, i0: int, i1: int) -> float:
        """0-based half-open range [i0, i1) == the reference's 1-based ``i0+1:i1`` (S:42-49)."""
        a = np.ascontiguousarray(a, dtype=np.float64)
        b = np.ascontiguousarray(b, dtype=np.float64)
        return float(self.lib.dhqr_oracle_partialdot(_fptr(a), _fptr(b), i0, i1))

    # -- qr! ------------------------------------------------------------------
    def qr(self, a: np.ndarray, nthreads: int = 0):
        """qr!(A::Matrix) (S:311-315): factor ``a`` in place, return (a, alpha)."""
        _check_colmajor(a)
        if nthreads <= 0:
            nthreads = min(self.max_threads(), 32)      # plenty for test sizes; bench.py passes its own count
        m, n = a.shape
        alpha = np.zeros(n)
        rc = self.lib.dhqr_oracle_qr(m, n, _fptr(a), a.strides[1] // 8 if n > 0 else max(m, 1), _fptr(alpha), nthreads)
        if rc:
            raise RuntimeError(f"dhqr_oracle_qr rc={rc}")
        return a, alpha

    def qr_steps(self, a: np.ndarray, jstop: int, nthreads: int = 0):
        _check_colmajor(a)
        m, n = a.shape
        alpha = np.zeros(n)
        fl = C.c_double(0.0)
        rc = self.lib.dhqr_oracle_qr_steps(m, n, _fptr(a), a.strides[1] // 8, _fptr(alpha), jstop, nthreads, C.byref(fl))
        if rc:
            raise RuntimeError(f"dhqr_oracle_qr_steps rc={rc}")
        return alpha, fl.value

    def qr_steps_strided(self, a: np.ndarray, j0: int, stride: int, nthreads: int = 0):
        """Column steps j0, j0+stride, ... of S:127-144 on the current contents of ``a`` (bench.py's bounded sample)."""
        _check_colmajor(a)
        m, n = a.shape
        alpha = np.zeros(n)
        fl = C.c_double(0.0)
        rc = self.lib.dhqr_oracle_qr_steps_strided(m, n, _fptr(a), a.strides[1] // 8, _fptr(alpha), j0, stride, nthreads,
                                                   C.byref(fl))
        if rc:
            raise RuntimeError(f"dhqr_oracle_qr_steps_strided rc={rc}")
        return alpha, fl.value

    @staticmethod
    def _blocks(blocks, col0s):
        arr = (_Block * len(blocks))()
        for k, (blk, c0) in enumerate(zip(blocks, col0s)):
            _check_colmajor(blk)
            arr[k] = _Block(blk.ctypes.data, blk.strides[1] // 8 if blk.shape[1] > 0 else max(blk.shape[0], 1), c0,
                            blk.shape[1])
        return arr

    def qr_blocks(self, m: int, n: int, blocks, col0s, nthreads: int = 0):
        """qr!(A::DArray) (S:115-119): ``blocks[p]`` is the localpart of owner p (m x n_p, col-major)."""
        alpha = np.zeros(n)
        arr = self._blocks(blocks, col0s)
        rc = self.lib.dhqr_oracle_householder_blocks(m, n, len(blocks), arr, _fptr(alpha), nthreads)
        if rc:
            raise RuntimeError(f"dhqr_oracle_householder_blocks rc={rc}")
        return alpha

    # -- solve ----------------------------------------------------------------
    def apply_qt(self, h: np.ndarray, b: np.ndarray) -> np.ndarray:
        _check_colmajor(h)
        m, n = h.shape
        w = np.array(b, dtype=np.float64, copy=True)
        self.lib.dhqr_oracle_apply_qt(m, n, _fptr(h), h.strides[1] // 8, _fptr(w))
        return w

    def backsolve(self, h: np.ndarray, alpha: np.ndarray, b: np.ndarray) -> np.ndarray:
        _check_colmajor(h)
        m, n = h.shape
        w = np.array(b, dtype=np.float64, copy=True)
        self.lib.dhqr_oracle_backsolve(m, n, _fptr(h), h.strides[1] // 8, _fptr(alpha), _fptr(w))
        return w[:n]

    def ldiv(self, h: np.ndarray, alpha: np.ndarray, b: np.ndarray) -> np.ndarray:
        """H \\ b (S:317-321)."""
        _check_colmajor(h)
        m, n = h.shape
        b = np.ascontiguousarray(b, dtype=np.float64)
        x = np.zeros(n)
        rc = self.lib.dhqr_oracle_ldiv(m, n, _fptr(h), h.strides[1] // 8, _fptr(alpha), _fptr(b), _fptr(x))
        if rc:
            raise RuntimeError(f"dhqr_oracle_ldiv rc={rc}")
        return x

    def solve_blocks(self, m, n, blocks, col0s, alpha, b):
        w = np.array(b, dtype=np.float64, copy=True)
        arr = self._blocks(blocks, col0s)
        self.lib.dhqr_oracle_solve_blocks(m, n, len(blocks), arr, _fptr(alpha), _fptr(w))
        return w[:n]

    def apply_qt_blocks(self, m, n, blocks, col0s, b):
        w = np.array(b, dtype=np.float64, copy=True)
        arr = self._blocks(blocks, col0s)
        self.lib.dhqr_oracle_apply_qt_blocks(m, n, len(blocks), arr, _fptr(w))
        return w

    # -- synthetic inputs -----------------------------------------------------
    def fill_uniform(self, seed: int, m: int, n: int, i0: int = 0, j0: int = 0) -> np.ndarray:
        a = np.empty((m, n), dtype=np.float64, order="F")
        self.lib.dhqr_oracle_fill_uniform(seed, i0, j0, m, n, _fptr(a), max(m, 1))
        return a


# ---------------------------------------------------------------------------
# numpy twin (independent restatement; small cases)
# ---------------------------------------------------------------------------
def np_alphafactor(x: float) -> float:
    """S:8."""
    return -float(np.sign(x))


def np_partialdot(a, b, i0, i1) -> float:
    """S:42-49 (0-based half-open)."""
    return float(np.dot(a[i0:i1], b[i0:i1]))


def np_qr(a: np.ndarray):
    """S:122-148 + S:198-213, single block.  Returns (H, alpha) without touching ``a``."""
    h = np.array(a, dtype=np.float64, order="F", copy=True)
    m, n = h.shape
    alpha = np.zeros(n)
    for j in range(n):
        s = np.linalg.norm(h[j:, j])                      # S:129
        alpha[j] = s * np_alphafactor(h[j, j])            # S:130
        f = 1.0 / np.sqrt(s * (s + abs(h[j, j])))         # S:131
        h[j, j] -= alpha[j]                               # S:132
        h[j:, j] *= f                                     # S:133-135
        hj = h[:, j].copy()                               # S:138-140
        if j + 1 < n:
            s_all = hj[j:] @ h[j:, j + 1:]                # S:208 for every jj
            h[j:, j + 1:] -= np.outer(hj[j:], s_all)      # S:209
    return h, alpha


def np_apply_qt(h, b):
    """S:232-242."""
    m, n = h.shape
    w = np.array(b, dtype=np.float64, copy=True)
    for j in range(n):
        s = h[j:, j] @ w[j:]
        w[j:] -= h[j:, j] * s
    return w


def np_backsolve(h, alpha, b):
    """S:244-254 / S:256-282."""
    m, n = h.shape
    w = np.array(b, dtype=np.float64, copy=True)
    for i in range(n - 1, -1, -1):
        w[i] = (w[i] - h[i, i + 1:n] @ w[i + 1:n]) / alpha[i]
    return w[:n]


def np_ldiv(h, alpha, b):
    """S:317-321."""
    return np_backsolve(h, alpha, np_apply_qt(h, b))


# ---------------------------------------------------------------------------
# ComplexF64 restatement (SURVEY section 8f "next": oracle first; no CUDA path yet)
# ---------------------------------------------------------------------------
def np_alphafactor_c(x: complex) -> complex:
    """S:9: alphafactor(x::Complex) = -exp(im * angle(x))   (angle(0) = 0 -> -1)."""
    return -np.exp(1j * np.angle(x))


def np_partialdot_c(a, b, i0, i1) -> complex:
    """S:51-59: sum conj(a[i]) * b[i]   (re = ar*br + ai*bi, im = ar*bi - ai*br)."""
    return complex(np.vdot(a[i0:i1], b[i0:i1]))


def np_qr_c(a: np.ndarray):
    """S:122-148 + S:198-213 for ComplexF64: H_j = I - v_j v_j^H with |v_j|^2 = 2, alpha_j = -exp(i angle(h_jj)) * norm."""
    h = np.array(a, dtype=np.complex128, order="F", copy=True)
    m, n = h.shape
    alpha = np.zeros(n, dtype=np.complex128)
    for j in range(n):
        s = np.linalg.norm(h[j:, j])                      # S:129
        alpha[j] = s * np_alphafactor_c(h[j, j])          # S:130
        f = 1.0 / np.sqrt(s * (s + abs(h[j, j])))         # S:131 (real)
        h[j, j] -= alpha[j]                               # S:132
        h[j:, j] *= f                                     # S:133-135
        hj = h[:, j].copy()                               # S:138-140
        if j + 1 < n:
            s_all = np.conj(hj[j:]) @ h[j:, j + 1:]       # S:208 with the complex partialdot (S:51-59)
            h[j:, j + 1:] -= np.outer(hj[j:], s_all)      # S:209 / S:162-196 (hotloop!: Hl -= Hj * s)
    return h, alpha


def np_apply_qt_c(h, b):
    """S:232-242 with the complex partialdot."""
    m, n = h.shape
    w = np.array(b, dtype=np.complex128, copy=True)
    for j in range(n):
        s = np.vdot(h[j:, j], w[j:])
        w[j:] -= h[j:, j] * s
    return w


def np_backsolve_c(h, alpha, b):
    """S:244-254 (no conjugation: plain triangular solve with diag(R) = alpha)."""
    m, n = h.shape
    w = np.array(b, dtype=np.complex128, copy=True)
    for i in range(n - 1, -1, -1):
        w[i] = (w[i] - h[i, i + 1:n] @ w[i + 1:n]) / alpha[i]
    return w[:n]


def np_ldiv_c(h, alpha, b):
    """S:317-321."""
    return np_backsolve_c(h, alpha, np_apply_qt_c(h, b))


def reconstruct_c(h, alpha):
    """Q R from the complex storage format: R = triu(H,1) + diag(alpha), Q = H_1 ... H_n."""
    m, n = h.shape
    r = np.zeros((m, n), dtype=np.complex128)
    r[:n] = np.triu(h[:n], 1) + np.diag(alpha)
    for j in range(n - 1, -1, -1):
        v = h[j:, j]
        r[j:] -= np.outer(v, np.conj(v) @ r[j:])
    return r


def np_uniform(seed: int, m: int, n: int, i0: int = 0, j0: int = 0) -> np.ndarray:
    """numpy twin of dhqr_oracle_fill_uniform (counter-based U[0,1) keyed on (seed, i, j))."""
    def mix(z):
        z = (z + np.uint64(0x9E3779B97F4A7C15))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))
    with np.errstate(over="ignore"):
        i = (np.arange(m, dtype=np.uint64) + np.uint64(i0))[:, None]
        j = (np.arange(n, dtype=np.uint64) + np.uint64(j0))[None, :]
        s = mix(np.array(seed, dtype=np.uint64))
        z = mix(s ^ (j * np.uint64(0xD1342543DE82EF95) + i))
    return np.asfortranarray((z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53)


# ---------------------------------------------------------------------------
# LAPACK comparator in the reference's storage format
# ---------------------------------------------------------------------------
def lapack_qr_refformat(a: np.ndarray):
    """dgeqrf -> (H, alpha) in the reference's format (SURVEY App. A)."""
    from scipy.linalg import lapack
    qr, tau, _, info = lapack.dgeqrf(np.asfortranarray(a))
    assert info == 0
    m, n = qr.shape
    h = np.asfortranarray(qr.copy())
    alpha = np.diag(qr)[:n].copy()
    for j in range(n):
        # v_ref = f*(x - alpha e1) carries the sign of the pivot x_j = -sign(alpha_j); LAPACK's v has v[0]=1
        st = -np.sign(alpha[j]) * np.sqrt(tau[j])
        h[j + 1:, j] = qr[j + 1:, j] * st
        h[j, j] = st
    return h, alpha


def lapack_lstsq(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """x = qr(A) \\ b through LAPACK — the reference tests' own oracle (T:49)."""
    from scipy.linalg import lapack, solve_triangular
    qr, tau, _, info = lapack.dgeqrf(np.asfortranarray(a))
    assert info == 0
    n = a.shape[1]
    cq, _, info = lapack.dormqr("L", "T", qr, tau, np.asfortranarray(b.reshape(-1, 1)), max(1, 64 * n))
    assert info == 0
    return solve_triangular(qr[:n, :n], cq[:n, 0], lower=False)


# ---------------------------------------------------------------------------
# metrics shared by the parity tests
# ---------------------------------------------------------------------------
def reconstruct(h: np.ndarray, alpha: np.ndarray) -> np.ndarray:
    """Q*R from the reference's storage format: R = triu(H,1) + diag(alpha); Q = H_1 ... H_n."""
    m, n = h.shape
    r = np.zeros((m, n))
    r[:n, :] = np.triu(h[:n, :], 1) + np.diag(alpha)
    nb = 64
    for k in range(((n - 1) // nb) * nb, -1, -nb):       # Q R = H_1 (H_2 (... H_n R)), blocked
        kb = min(nb, n - k)
        v = np.tril(h[k:, k:k + kb])
        s = v.T @ v
        linv_t = np.linalg.inv(np.eye(kb) + np.tril(s, -1)).T   # T = (I + striu(V'V))^-1
        r[k:, :] -= v @ (linv_t @ (v.T @ r[k:, :]))
    return r


def qr_residual(a0: np.ndarray, h: np.ndarray, alpha: np.ndarray) -> float:
    """||QR - A||_F / ||A||_F (BASELINE.json metric)."""
    return float(np.linalg.norm(reconstruct(h, alpha) - a0) / np.linalg.norm(a0))


def normal_eq_residual(a: np.ndarray, x: np.ndarray, b: np.ndarray) -> float:
    """||A'A x - A'b||_2 — the reference's only assertion (T:51, T:62, T:81)."""
    return float(np.linalg.norm(a.T @ (a @ x) - a.T @ b))
