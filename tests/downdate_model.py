"""numpy restatement of the device's downdate (dhqr_qr_downdate_f64 / dhqr_apply_downdate_f64, DESIGN §2.11): Theta [R; Z] = [R'; 0]
with R''R' = R'R - Z'Z, in the structure of append_model.py (outer panels of 128 columns, each four 32-column panels factored
column by column with the 32-wide block update of the rest of the outer panel after each, then the 128-wide block update of the
trailing columns), with hyperbolic reflectors Theta_j = I - v~_j v~_j' J, J = diag(I_n, -I_k), v~_j' J v~_j = 2 (or 0).

Storage as on the device: R is an (n, n) array whose strict upper triangle is R's, alpha = diag(R); Z (k, n) is overwritten with
the reflector tails V2; vtop[j] sits on row j of the R block.  The first column with sigma^2 <= 0 while t > 0, or a NaN sigma^2,
fails: info is its 1-based index, and it and every later column store vtop = 0, V2 = 0, alpha = NaN.

ext_downdate runs the unblocked recurrence in long double (tests/downdate_ext.c, compiled on first use into a temporary directory
as tests/adjoint_oracle.py does)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

NB, IB = 128, 32
_HERE = os.path.dirname(os.path.abspath(__file__))


def _column(x0, t):
    """(sigma, alpha, f, vtop, fails) of one column from x0 = R[j, j] and t = ||Z[:, j]||^2."""
    rt, ax = np.sqrt(t), abs(x0)
    s2 = (ax - rt) * (ax + rt)
    fails = bool(np.isnan(s2) or (t > 0.0 and s2 <= 0.0))
    if fails:
        return 0.0, np.nan, 0.0, 0.0, True
    s = np.sqrt(s2)
    if s == 0.0:
        return 0.0, 0.0, 0.0, 0.0, False
    al = -s if x0 >= 0.0 else s                      # a zero x0 counts as positive
    f = 1.0 / np.sqrt(s * (s + ax))
    return s, al, f, f * (x0 - al), False


def _panel(R, alpha, Z, vtop, j0, nc, st):
    for j in range(j0, j0 + nc):
        t = Z[:, j] @ Z[:, j:j0 + nc]                # the exchanged totals: Z[:, j]' Z[:, c], c >= j
        _, al, f, vt, fails = _column(alpha[j], t[0])
        if st["info"] or fails:
            st["info"] = st["info"] or j + 1
            Z[:, j] = 0.0
            alpha[j], vtop[j] = np.nan, 0.0
            continue
        w = vt * R[j, j + 1:j0 + nc] - f * t[1:]
        R[j, j + 1:j0 + nc] -= vt * w
        Z[:, j] *= f
        Z[:, j + 1:j0 + nc] -= np.outer(Z[:, j], w)
        alpha[j], vtop[j] = al, vt


def _block(V2, vt, X, C):
    """[X; C] <- Theta_blk [X; C] for V~ = [diag(vt); V2]: W = diag(vt) X - V2' C, T^{-1} = I - striu(V2'V2), Y = -T'W."""
    if X.shape[1] == 0:
        return
    W = vt[:, None] * X - V2.T @ C
    T = np.linalg.inv(np.eye(V2.shape[1]) - np.triu(V2.T @ V2, 1))
    Y = -T.T @ W
    C += V2 @ Y
    X += vt[:, None] * Y


def qr_downdate(R, alpha, Z):
    """Returns (R, alpha, V2, vtop, info): copies, R' in R's strict upper triangle and alpha."""
    R, alpha, Z = np.array(R, dtype=float), np.array(alpha, dtype=float), np.array(Z, dtype=float)
    n = alpha.size
    vtop = np.zeros(n)
    st = {"info": 0}
    for k0 in range(0, n, NB):
        kb = min(NB, n - k0)
        for o in range(0, kb, IB):
            cs, w = k0 + o, min(IB, kb - o)
            _panel(R, alpha, Z, vtop, cs, w, st)
            _block(Z[:, cs:cs + w], vtop[cs:cs + w], R[cs:cs + w, cs + w:k0 + kb], Z[:, cs + w:k0 + kb])
        _block(Z[:, k0:k0 + kb], vtop[k0:k0 + kb], R[k0:k0 + kb, k0 + kb:], Z[:, k0 + kb:])
    return R, alpha, Z, vtop, st["info"]


def apply_downdate(V2, vtop, c, e):
    """[c; e] <- Theta [c; e] block by block, first to last, as the device does; returns copies."""
    c, e = np.array(c, dtype=float), np.array(e, dtype=float)
    for o in range(0, vtop.size, NB):
        kb = min(NB, vtop.size - o)
        _block(V2[:, o:o + kb], vtop[o:o + kb], c[o:o + kb], e)
    return c, e


def unblocked(R, alpha, Z, c=None, e=None):
    """The column recurrence of the issue, one reflector at a time: (R, alpha, V2, vtop, info[, c', e'])."""
    R, alpha, Z = np.array(R, dtype=float), np.array(alpha, dtype=float), np.array(Z, dtype=float)
    n = alpha.size
    vtop, info = np.zeros(n), 0
    rhs = c is not None
    if rhs:
        c, e = np.array(c, dtype=float), np.array(e, dtype=float)
    for j in range(n):
        _, al, f, vt, fails = _column(alpha[j], Z[:, j] @ Z[:, j])
        if info or fails:
            info = info or j + 1
            Z[:, j] = 0.0
            alpha[j], vtop[j] = np.nan, 0.0
            continue
        Z[:, j] *= f
        w = vt * R[j, j + 1:] - Z[:, j] @ Z[:, j + 1:]
        R[j, j + 1:] -= vt * w
        Z[:, j + 1:] -= np.outer(Z[:, j], w)
        alpha[j], vtop[j] = al, vt
        if rhs:
            wc = vt * c[j] - Z[:, j] @ e
            c[j] -= vt * wc
            e -= np.outer(Z[:, j], wc)
    return (R, alpha, Z, vtop, info) + ((c, e) if rhs else ())


_lib = None


def _load():
    global _lib
    if _lib is None:
        out = tempfile.mkdtemp(prefix="downdate_ext_")
        so = os.path.join(out, "libdowndate_ext.so")
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else (shutil.which("gcc") or "cc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-shared", "-o", so, os.path.join(_HERE, "downdate_ext.c"), "-lm"])
        _lib = C.CDLL(so)
        _lib.downdate_ext.restype = C.c_int64
        _lib.downdate_ext.argtypes = [C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int64]
    return _lib


def ext_downdate(R, alpha, Z, c=None, e=None):
    """unblocked() in long double, rounded to double when written out: (R, alpha, V2, vtop, info[, c', e'])."""
    n, k = alpha.size, Z.shape[0]
    Rf = np.asfortranarray(np.array(R, dtype=float))
    a = np.array(alpha, dtype=float)
    Zf = np.asfortranarray(np.array(Z, dtype=float))
    vt = np.zeros(n)
    rhs = c is not None
    cf = np.asfortranarray(np.array(c, dtype=float).reshape(n, -1)) if rhs else np.zeros((n, 0), order="F")
    ef = np.asfortranarray(np.array(e, dtype=float).reshape(k, -1)) if rhs else np.zeros((k, 0), order="F")
    p = lambda t: C.c_void_p(t.ctypes.data) if t.size else None
    info = _load().downdate_ext(n, k, p(Rf), p(a), p(Zf), p(vt), p(cf), p(ef), cf.shape[1])
    out = (Rf, a, Zf, vt, int(info))
    if rhs:
        out += (cf.reshape(np.shape(c)), ef.reshape(np.shape(e)))
    return out
