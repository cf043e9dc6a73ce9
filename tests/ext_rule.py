"""The extended-precision acceptance rule shared by the GPU accuracy modules (test_gpu_ext.py: every path on hard families;
test_gpu_shapes.py: the same rule at the shape edges; test_gpu_complex_ext.py: every ComplexF64 path on the complex families).

The reference is oracle/dhqr_oracle.c's loop in long double (COracle.qr_ext): the reference's recurrences with a forward error
of about kappa * 1e-19.  The fp64 oracle runs the same loop in double, so its error against the extended reference on the
same input is what the reference algorithm in the reference's precision achieves.  The library is held to that:

    err_gpu <= C_REL * max(err_fp64_oracle, FLOOR)        for each metric below

Metrics (all against the extended reference; tests/matrix_families.py has the inputs):
    V     max |dH| over the lower trapezoid (the reflectors, entries O(1) since |v|^2 = 2)
    R     max |dR_ij| / ||A[:, j]|| over the strict upper triangle and alpha (column-relative: R spans 10^+-120 in colscale)
    qtb   ||d(Q'b)|| / ||b||          qb  ||d(Qb)|| / ||b||          x   ||dx|| / ||x||
FLOOR = 16 eps for V and R, 16 eps sqrt(m) for the solve metrics.  Two absolute bounds on every family inside the reference's
range:
    bwd   max_j ||(QR - A)[:, j]|| / ||A[:, j]|| < 1e-13
    orth  max_j | ||v_j||^2 - 2 | < 1e-13
"""
import contextlib
import hashlib
import os

import numpy as np
import torch

import matrix_families as F

EPS = np.finfo(np.float64).eps
C_REL = 8            # headroom over the fp64 oracle: the blocked paths sum in other orders (split-K, CholeskyQR2 + reconstruction)
# Where the floor decides, the margin is thinnest: on triangular input the oracle's reflectors are +-sqrt(2) e_j to an ulp, while
# the blocked update still rounds every R entry once per 128-column panel to its left and in its split-K sums.  Measured on an
# H100 SXM (132 SMs): R error 98 eps (ratio 6.1) at 4099 x 640, 1.5 at 2048 x 1024; every non-triangular cell <= 1.5.  Split
# counts follow the SM count, so a part with other SMs moves this cell first; a ratio near 8 there is summation order, not a bug.
FLOOR_EPS = 16       # FLOOR = 16 eps x size factor: for inputs where the fp64 oracle happens to be (nearly) exact, e.g. triangular
SIZE = {"V": lambda m: 1.0, "R": lambda m: 1.0,            # one rounded result of a stable recurrence per entry: the oracle lands at 1-4 eps
        "qtb": np.sqrt, "qb": np.sqrt, "x": np.sqrt}        # a sweep over m rows: rounding errors add up like a random walk
TOL_BWD = 1e-13      # column-wise backward error: Householder QR is column-wise backward stable whatever kappa is
TOL_ORTH = 1e-13     # |v_j|^2 = 2 exactly in exact arithmetic (S:131-135)
COUNTERS = ("wide_panels", "wide_redone", "panels_fast", "panels_fallback")
RHS = 4              # default right-hand-side block of a real Ref: column 0 the single right-hand side, 1..3 an nrhs = 3 block
# Ref.check_oracles_agree: err_fp64 <= AGREE kappa eps.  Worst measured on the complex families at 1024 x 384 and 777 x 321:
# 781 kappa eps (imag: a pivot whose real part is exactly 0 in extended precision and rounding in fp64, divided by a pivot
# 6e-4 of its column's norm); an oracle pair that disagrees on a convention is off by O(1)
AGREE = 4096


@contextlib.contextmanager
def options(h, **kw):
    """Set options on a handle for the duration of a block and put back what was there.  A profiled block drains the per-launch
    CUDA-event brackets it left on the handle."""
    prev = {k: h.get_option(k) for k in kw}
    try:
        for k, v in kw.items():
            h.set_option(k, v)
        yield h
    finally:
        for k, v in prev.items():
            h.set_option(k, v)
        if kw.get("profile"):
            h.profile_reset()


def counters(h):
    return {k: h.get_option(k) for k in COUNTERS}


# ---------------------------------------------------------------------------------------------------------------------
# references: one extended + one fp64 computation per input
# ---------------------------------------------------------------------------------------------------------------------
def nrm(v):
    s = float(np.nanmax(np.abs(v))) if np.size(v) else 0.0
    return s * float(np.linalg.norm(v / s)) if s > 0 and np.isfinite(s) else s


def qb_sweep(h, b):
    w = np.array(b, dtype=h.dtype, copy=True)
    for j in range(h.shape[1] - 1, -1, -1):
        w[j:] -= h[j:, j] * (h[j:, j] @ w[j:])
    return w


class Ref:
    """Extended and fp64 results for one input.  ``k`` leading columns are compared (the leading-column identity: H[:, :k] and
    alpha[:k] depend on A[:, :k] only); for the zero-column families k is the zero column, and the NaN pattern of the whole
    fp64 oracle (COracle.qr, or np_qr_c for complex input) is kept for comparison.

    ``nrhs`` right-hand sides (default: RHS for real input, one length-m vector for complex) go through both references;
    b, qtb_e, qb_e, x_e, qtb64, qb64 and x64 are then (m or n, nrhs) blocks, except for the complex single vector.  Solves are
    skipped (``solve`` False) for the zero-column families and where the family is singular at the shape (F.singular), for
    real and complex input alike."""

    def __init__(self, coracle, oracle, family, m, n, k=None, cplx=False, solve=True, nrhs=None, keep_h64=False):
        self.family, self.m, self.n = family, m, n
        A = F.make_complex(family, m, n) if cplx else F.make(family, m, n)
        self.A = A
        self.nan_cols = self.nan_alpha = None
        if family in (F.COMPLEX_NAN_FAMILIES if cplx else F.NAN_FAMILIES):
            with np.errstate(all="ignore"):
                H64, a64 = oracle.np_qr_c(A) if cplx else coracle.qr(A.copy(order="F"))
            self.nan_cols, self.nan_alpha = np.isnan(H64).any(0), np.isnan(a64)
            k, solve = F.zero_column(family, n), False
        k = n if k is None else k
        solve = solve and not F.singular(family, m, k)
        self.k, self.solve = k, solve
        Ak = np.asfortranarray(A[:, :k])
        self.cn = np.linalg.norm(Ak, axis=0)
        if cplx and not solve:
            self.He, self.ae = coracle.qr_ext_c(Ak)
            self.H64, self.a64 = oracle.np_qr_c(Ak)
        elif cplx and nrhs is None:
            self.b = F.rhs(m, 1, cplx=True)
            self.He, self.ae, qtb, x = coracle.qr_ext_c(Ak, self.b)
            self.qtb_e, self.x_e = qtb[:, 0], x[:, 0]
            self.H64, self.a64 = oracle.np_qr_c(Ak)
            self.qtb64 = oracle.np_apply_qt_c(self.H64, self.b)
            self.x64 = oracle.np_ldiv_c(self.H64, self.a64, self.b)
        elif cplx:
            self.b = np.asfortranarray(F.rhs(m, nrhs, cplx=True).reshape(m, nrhs))
            self.He, self.ae, self.qtb_e, self.x_e = coracle.qr_ext_c(Ak, self.b)
            self.H64, self.a64 = oracle.np_qr_c(Ak)
            self.qtb64 = np.stack([oracle.np_apply_qt_c(self.H64, self.b[:, r]) for r in range(nrhs)], 1)
            self.x64 = np.stack([oracle.np_ldiv_c(self.H64, self.a64, self.b[:, r]) for r in range(nrhs)], 1)
        elif solve:
            nrhs = RHS if nrhs is None else nrhs
            self.b = np.asfortranarray(F.rhs(m, nrhs).reshape(m, nrhs))
            self.He, self.ae, self.qtb_e, self.qb_e, self.x_e = coracle.qr_ext(Ak, self.b, want_qb=True)
            self.H64, self.a64 = coracle.qr(Ak.copy(order="F"))
            self.qtb64 = np.stack([coracle.apply_qt(self.H64, self.b[:, r].copy()) for r in range(nrhs)], 1)
            self.qb64 = np.stack([qb_sweep(self.H64, self.b[:, r]) for r in range(nrhs)], 1)
            self.x64 = np.stack([coracle.ldiv(self.H64, self.a64, self.b[:, r].copy()) for r in range(nrhs)], 1)
        else:
            self.He, self.ae = coracle.qr_ext(Ak)
            self.H64, self.a64 = coracle.qr(Ak.copy(order="F"))
        self.e64 = factor_errors(self.H64, self.a64, self)
        if not keep_h64:
            del self.H64                                 # only its errors (and solves, above) are needed from here on

    def check_oracles_agree(self, c=AGREE):
        """Both oracles describe the same factorisation: err_fp64 <= c kappa eps on V and R, kappa the 2-norm condition number
        of the leading columns scaled to unit norm.  A convention on which the two differ (the phase of a zero pivot, say)
        makes err_fp64 O(1), and every rule measured against it would pass whatever the library returns."""
        Ak = self.A[:, :self.k] / np.where(self.cn > 0, self.cn, 1.0)
        kappa = float(np.linalg.cond(Ak))
        for key in ("V", "R"):
            assert self.e64[key] <= c * kappa * EPS, \
                f"the fp64 and extended oracles disagree on {key}: {self.e64[key]:.3e} > {c} x kappa {kappa:.3e} x eps; " \
                f"family {self.family}, {self.m}x{self.n}"
        return kappa

    def solve_errors(self, key, got, r):
        """(err_gpu, err_fp64) of right-hand side ``r`` for metric ``key`` in qtb, qb, x; ``got`` is the library's result."""
        e, e64 = getattr(self, key + "_e"), getattr(self, key + "64")
        scale = nrm(self.x_e[:, r]) if key == "x" else nrm(self.b[:, r])
        return nrm(got - e[:, r]) / scale, nrm(e64[:, r] - e[:, r]) / scale


# ---------------------------------------------------------------------------------------------------------------------
# metrics and the acceptance rule
# ---------------------------------------------------------------------------------------------------------------------
def factor_errors(H, alpha, ref):
    k = ref.k
    dH = H[:, :k] - ref.He
    with np.errstate(all="ignore"):
        return {"V": float(np.abs(np.tril(dH)).max()),
                "R": float(max((np.abs(np.triu(dH[:k], 1)) / ref.cn).max(), (np.abs(alpha[:k] - ref.ae) / ref.cn).max()))}


def orth_error(H, k):
    v = np.tril(H[:, :k])
    return float(np.abs((np.abs(v) ** 2).sum(0) - 2.0).max())


def backward_error(A0, H, alpha, dev="cuda:0"):
    """max_j ||(QR - A)[:, j]|| / ||A[:, j]||, formed on the GPU in fp64.  Columns are first scaled by a power of two near their
    norm (exact), so 1e-150 or 1e+-120 columns neither underflow nor overflow in the residual."""
    m, k = A0.shape
    cn = np.linalg.norm(A0, axis=0)
    p = np.ldexp(1.0, np.round(np.log2(np.where(cn > 0, cn, 1.0))).astype(int))
    A = torch.from_numpy(np.ascontiguousarray(A0 / p)).to(dev)
    Hd = torch.from_numpy(np.ascontiguousarray(H[:, :k])).to(dev)
    al = torch.from_numpy(np.ascontiguousarray(alpha[:k]))
    R = torch.zeros(m, k, dtype=A.dtype, device=dev)
    R[:k] = torch.triu(Hd[:k], 1) + torch.diag(al.to(dev))
    R /= torch.from_numpy(p).to(dev)
    for c in range(((k - 1) // 128) * 128, -1, -128):
        kb = min(128, k - c)
        V = torch.tril(Hd[c:, c:c + kb])
        Tinv = torch.eye(kb, dtype=A.dtype, device=dev) + torch.triu(V.mH @ V, 1)
        R[c:] -= V @ torch.linalg.solve_triangular(Tinv, V.mH @ R[c:], upper=True)
    return float(((R - A).norm(dim=0) / A.norm(dim=0)).max())


class Table:
    """The worst ratio err_gpu / max(err_fp64_oracle, FLOOR) per (path, family), written to build/<name> when a module ends,
    plus the wide chain's counters per factorisation where a module records them."""

    def __init__(self, name):
        self.name = name
        self.ratios = {}
        self.counts = {}

    def check(self, path, ref, gpu, e64, absolute=None, note="", c_rel=C_REL):
        """The relative rule on every metric in ``gpu`` (err_gpu <= c_rel max(err_fp64, FLOOR)) and the absolute bounds."""
        floor = {key: FLOOR_EPS * EPS * SIZE[key](ref.m) for key in gpu}
        worst = max(((gpu[key] / max(e64[key], floor[key]), key) for key in gpu), key=lambda t: (np.nan_to_num(t[0], nan=np.inf), t[1]))
        prev = self.ratios.get((path, ref.family))
        if prev is None or np.nan_to_num(worst[0], nan=np.inf) > np.nan_to_num(prev[0], nan=np.inf):
            self.ratios[(path, ref.family)] = worst
        where = f"path {path}, family {ref.family}, {ref.m}x{ref.n}; {note}"
        for key in gpu:
            assert gpu[key] <= c_rel * max(e64[key], floor[key]), \
                f"{key}: err_gpu {gpu[key]:.3e} > {c_rel} x max(err_fp64 {e64[key]:.3e}, floor {floor[key]:.1e}); {where}"
        for key, (val, tol) in (absolute or {}).items():
            assert val < tol, f"{key} = {val:.3e} >= {tol:.0e}; {where}"

    def write(self):
        if not self.ratios:
            return
        paths = list(dict.fromkeys(p for p, _ in self.ratios))
        fams = list(dict.fromkeys(f for _, f in self.ratios))
        lines = ["# err_gpu / max(err_fp64_oracle, FLOOR), worst metric per cell (rule: <= %d)" % C_REL, "",
                 "| path | " + " | ".join(fams) + " |", "|---|" + "---|" * len(fams)]
        tail = ["", "wide chain per factorisation: (panels it factored, restarts after a refusal)", ""] + \
            [f"- {p} {f}: {c}" for (p, f), c in self.counts.items()]
        for p in paths:
            cells = []
            for f in fams:
                r = self.ratios.get((p, f))
                cells.append("" if r is None else f"{r[0]:.2g} {r[1]}")
            lines.append(f"| {p} | " + " | ".join(cells) + " |")
        try:
            out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build")
            os.makedirs(out, exist_ok=True)
            with open(os.path.join(out, self.name), "w") as fh:
                fh.write("\n".join(lines + tail) + "\n")
        except OSError:
            pass


def run_qr(D, A0, nb=0, lda_extra=0, handle=None, **opts):
    h = handle or D.default_handle(0)
    m, n = A0.shape
    with options(h, **opts):
        c0 = counters(h)
        dA = D.colmajor_empty(m, n, "cuda:0", lda=m + lda_extra, dtype=torch.from_numpy(A0[:1, :1]).dtype)
        dA.copy_(torch.from_numpy(A0))
        st = D.qr_(dA, nb=nb, handle=h)
        torch.cuda.synchronize()
        c1 = counters(h)
    note = "counters " + ", ".join(f"{k} {c0[k]}->{c1[k]}" for k in COUNTERS)
    return dA, st, note, {k: c1[k] - c0[k] for k in COUNTERS}


def check_nan_pattern(path, ref, H, alpha, note):
    where = f"path {path}, family {ref.family}, {ref.m}x{ref.n}; {note}"
    assert np.array_equal(np.isnan(H).any(0), ref.nan_cols), f"NaN columns differ from the fp64 oracle's; {where}"
    assert np.array_equal(np.isnan(alpha), ref.nan_alpha), f"NaN entries of alpha differ from the fp64 oracle's; {where}"
    assert np.isfinite(H[:, :ref.k]).all() and np.isfinite(alpha[:ref.k]).all(), where


def factor_checks(path, ref, H, alpha, note):
    if ref.nan_cols is not None:
        check_nan_pattern(path, ref, H, alpha, note)
    k = ref.k
    gpu = factor_errors(H, alpha, ref)
    absolute = {"bwd": (backward_error(np.asfortranarray(ref.A[:, :k]), H, alpha), TOL_BWD), "orth": (orth_error(H, k), TOL_ORTH)}
    return gpu, absolute


def digest(*arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in arrays)).hexdigest()
