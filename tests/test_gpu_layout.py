"""Storage contract of every entry point (run with -m gpu on an H100): results are bitwise independent of the leading dimension
and of the base address, nothing outside the m x n operand is written, and nothing outside it is read into a result.

Four kernels choose how to move an operand from its address and leading dimension; none of those choices changes the arithmetic
(the same values land in the same shared-memory slots), so the output must not change in a single bit:

    k_gemm_cvy_p   C tiles by bulk copies when C is 16 B aligned and ldc is even (rows at an odd end of a column's bulk segment
                   by generic loads and stores), otherwise 8-byte cp.async fills and generic stores
    k_gemm_vta     the A columns of V'[V | C] by bulk copies when C is 16 B aligned and ldc is even (a_aligned), else generic
    k_pack         double2 loads when A is 16 B aligned, lda is even and the window top is a multiple of 4, else scalar loads
    k_apply1_tma   (nb = 1) the columns by TMA when the window start is 16 B aligned and lda is even (aligned), else generic

Every operand window those kernels see starts at an even row of the operand (32-row aligned panel windows; row j - lead of
nb = 1), so the branch follows from the layout of the operand alone.  "Fast" below is bulk C tiles in k_gemm_cvy_p, bulk A
columns in k_gemm_vta, double2 loads in k_pack and TMA columns in k_apply1_tma; "generic" is the cp.async fill with generic
stores, the generic fill, scalar loads and the generic fill.  Each layout is compared with L0, the plain colmajor_empty operand:

    layout  ld                          base      branches
    L0      m                           16 B      fast when m is even; generic when m is odd (odd ld)
    L1      even, >= m + 2              16 B      fast, lda padding rows present; at odd m the odd last row of every column's
                                                  bulk segment in k_gemm_cvy_p (and the odd tail row of k_gemm_vta / k_apply1_tma)
                                                  moves by generic loads and stores
    L2      even, >= m + 2, r0 = 1      8 B off   generic with an even stride (every Julia view(B, 2:m+1, :) of an even-height B)
    L3      odd, >= m + 1               16 B      generic; every other column start is 16 B aligned
    L4      odd, >= m + 1               8 B off   generic
    L5      m + 67, r0 = 2 rows above,  16 B      a block of a larger matrix: fast when m + 67 is even (m odd), generic when
            2 guard columns each side             it is odd (m even)

So at m = 2050 L0 runs the fast branches against the generic ones of L2..L4, and at m = 1537 the generic ones against the fast
ones of L1 and L5.  The right-hand sides of the solves are the C operand of the same kernels (apply_qt / apply_q with nrhs > 1,
form_q's Q) or the vector of the GEMV sweep and the back-substitution, in the same kinds of layout.  ComplexF64 is moved as its
real view, which has an even stride and is 16 B aligned at any complex element offset, so the invariance holds trivially there
and any difference is a bug.

Guarded operands: every operand lives in a larger buffer whose other elements all hold one NaN bit pattern (SENTINEL).  After
every call each of them must still hold exactly that pattern (compared as int64: a NaN the library computed has other bits), so
a stray write fails, and a stray read that feeds arithmetic turns a result into NaN, which fails the bitwise comparison.

One fresh handle for the module, its workspace grown first to the largest problem here: split-K counts follow the workspace
size, and every comparison must see the same splits.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from ext_rule import counters, options
from test_gpu_ext import PATHS

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SENTINEL = 0x7FF4DEADBEEF0001          # a signalling-NaN bit pattern no arithmetic produces
SHAPES = [(2050, 1000), (1537, 777)]   # m even / odd; ragged last outer (128) and inner (32) panels, >= 2 full wide panels
HOST_SHAPE = (2050, 1408)              # host_chunk = 512 still splits the upload (n >= 3 * 512 / 2 + 512)
WARM = (8600, 1408)                    # the largest m and n of the module


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="module")
def h(D):
    h = D.Handle(0)
    A = D.colmajor_empty(*WARM, DEV)
    D.fill_uniform_(A, 3, handle=h)
    D.qr_(A, handle=h)
    torch.cuda.synchronize()
    del A
    yield h
    torch.cuda.synchronize()
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# guarded operands
# ---------------------------------------------------------------------------------------------------------------------
class Guarded:
    """An m x n column-major operand with leading dimension ld at element offset g * ld + r0 of a buffer of (n + 2g) ld elements
    (g guard columns on each side, r0 rows above), every other element of which holds SENTINEL.  ``A`` is the operand view; a
    single column (``vec``) is its 1-D view.  Works on the device or in (pinned) host memory, for float64 and complex128."""

    def __init__(self, m, n, ld, r0=0, g=1, dtype=torch.float64, device=DEV, pin=False):
        assert ld >= max(m, 1) and 0 <= r0 <= ld and g >= 1
        self.m, self.n, self.ld, self.r0, self.g = m, n, ld, r0, g
        size = (n + 2 * g) * ld
        self.buf = torch.empty(size, dtype=dtype, pin_memory=True) if pin else torch.empty(size, dtype=dtype, device=device)
        self.words = self.buf.view(torch.int64)
        self.words.fill_(SENTINEL)
        self.off = g * ld + r0
        self.A = self.buf.as_strided((m, n), (1, ld), self.off)
        outside = torch.ones(size, dtype=torch.bool, device=self.buf.device)
        outside.as_strided((m, n), (1, ld), self.off).fill_(False)
        self.outside = outside.repeat_interleave(self.words.numel() // size)

    @property
    def vec(self):
        assert self.n == 1
        return self.A[:, 0]

    @property
    def aligned(self):
        return self.A.data_ptr() % 16 == 0

    def check(self, where):
        bad = (self.words != SENTINEL) & self.outside
        nbad = int(bad.sum())
        if nbad:
            i = int(bad.nonzero()[0, 0]) // (self.words.numel() // self.buf.numel())
            col, row = divmod(i - self.g * self.ld, self.ld)
            raise AssertionError(f"{nbad} words outside the operand changed, the first at buffer element {i} (operand row {row - self.r0}, "
                                 f"column {col}; ld {self.ld}, {self.r0} rows above, {self.g} guard columns); {where}")


def placed(m, n, ld, misaligned, g=1):
    """A guarded Float64 operand whose base is 16 B aligned or 8 B off one, whatever the parity of ld."""
    G = Guarded(m, n, ld, ((g * ld) & 1) ^ int(misaligned), g)
    assert G.aligned != misaligned
    return G


def layouts(m):
    """name -> (ld, r0, g) of the Float64 layouts L1..L5 (table in the module docstring)."""
    even, odd = m + 2 + (m & 1), m + 1 + (m & 1)
    return {"L1": (even, 0, 1), "L2": (even, 1, 1), "L3": (odd, 0, 2), "L4": (odd, 0, 1), "L5": (m + 67, 2, 2)}


ALIGNED = {"L1": True, "L2": False, "L3": True, "L4": False, "L5": True}


def guarded_layout(name, m, n):
    ld, r0, g = layouts(m)[name]
    G = Guarded(m, n, ld, r0, g)
    assert G.aligned == ALIGNED[name], name
    return G


def bits(t):
    t = t.contiguous()
    return t.view(torch.int64) if t.dim() else t.reshape(1).view(torch.int64)


def assert_bitwise(got, ref, where):
    a, b = bits(got), bits(ref)
    assert a.shape == b.shape, where
    ne = a != b
    if bool(ne.any()):
        idx = tuple(int(i) for i in ne.nonzero()[0])
        raise AssertionError(f"{int(ne.sum())} words differ from L0 in their bits, the first at {idx} (int64 view of "
                             f"{got.dtype}); {where}")


def matrix(seed, m, n, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(m, n, dtype=torch.float64, generator=g)
    if dtype == torch.complex128:
        A = torch.complex(A, torch.randn(m, n, dtype=torch.float64, generator=g))
    return A.to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# Float64 factorisation: every path in every layout
# ---------------------------------------------------------------------------------------------------------------------
BLOCKED = ("default", "wide_panel0", "nb32", "nb64", "nb96", "lookahead0", "panel_fast0")
FACTOR_CASES = [(p, m, n) for m, n in SHAPES for p in BLOCKED] + [
    # nb = 1: k_unblocked_wave (m <= 8192), and with unblocked_wave = 0 the fused k_house1 + k_apply1_tma chain
    ("nb1_m8192", 2050, 1000), ("nb1_m8192", 1537, 777), ("nb1_wave0", 2050, 1000), ("nb1_wave0", 1537, 777),
    # fused chain (8193 <= m <= 8531), per-column launches: k_apply1_direct for the first steps, then k_apply1_tma (m >= 8533)
    ("nb1_m8193", 8300, 130), ("nb1_m8193", 8301, 130), ("nb1_m8533", 8600, 96),
    # fuse_house = 0 above the wave's limit: k_house1 and k_apply1_tma launched separately for every column
    ("nb1_fuse0", 8300, 130)]


def factor(D, h, A, nb, alpha_guard=None):
    n = A.shape[1]
    alpha = alpha_guard.vec if alpha_guard is not None else torch.zeros(n, dtype=A.dtype, device=DEV)
    D.householder_(A, alpha, nb=nb, handle=h)
    torch.cuda.synchronize()
    return alpha


@pytest.mark.parametrize("path,m,n", FACTOR_CASES, ids=[f"{p}-{m}x{n}" for p, m, n in FACTOR_CASES])
def test_factorisation_is_bitwise_independent_of_the_layout(D, h, path, m, n):
    nb, opts = PATHS[path][2], PATHS[path][4]
    A0 = matrix(m + n, m, n)
    with options(h, **opts):
        H0 = D.colmajor_empty(m, n, DEV)
        H0.copy_(A0)
        a0 = factor(D, h, H0, nb)
        for name in layouts(m):
            G, ga = guarded_layout(name, m, n), Guarded(n, 1, n, 0, 1)
            G.A.copy_(A0)
            a = factor(D, h, G.A, nb, ga)
            where = f"path {path} ({opts}, nb {nb}), {m}x{n}, layout {name}"
            assert_bitwise(G.A, H0, "H: " + where)
            assert_bitwise(a, a0, "alpha: " + where)
            G.check("A: " + where)
            ga.check("alpha: " + where)


def test_restart_after_a_refused_panel_is_layout_independent(D, h):
    # a nearly dependent column pair in the second outer panel: the wide chain refuses it on the device and qr! redoes the
    # factorisation from there; the verdicts come from the same values in every layout
    m, n = 2050, 640
    A0 = matrix(11, m, n)
    A0[:, 200] = A0[:, 150] + 1e-11 * matrix(12, m, 1)[:, 0]
    c0 = counters(h)
    H0 = D.to_colmajor(A0, DEV)
    a0 = factor(D, h, H0, 0)
    c1 = counters(h)
    d0 = {k: c1[k] - c0[k] for k in ("wide_panels", "wide_redone")}
    assert d0["wide_redone"] >= 1 and d0["wide_panels"] >= 4, d0
    for name in layouts(m):
        G = guarded_layout(name, m, n)
        G.A.copy_(A0)
        c0 = counters(h)
        a = factor(D, h, G.A, 0)
        c1 = counters(h)
        d = {k: c1[k] - c0[k] for k in d0}
        assert d == d0, f"layout {name}: wide chain {d}, L0 {d0}"
        assert_bitwise(G.A, H0, f"H, layout {name}")
        assert_bitwise(a, a0, f"alpha, layout {name}")
        G.check(f"layout {name}")


# ---------------------------------------------------------------------------------------------------------------------
# solves on each layout of the factorisation, with b in guarded layouts too
# ---------------------------------------------------------------------------------------------------------------------
def solve_ops(D, h):
    """name -> (options, fn(b, A, alpha)).  Every op overwrites b in place; all m rows of b are compared."""
    return {
        "apply_qt qt_vec=1": ({"qt_vec": 1}, lambda b, A, al: D.apply_qt_(b, A, h)),
        "apply_qt qt_vec=0": ({"qt_vec": 0}, lambda b, A, al: D.apply_qt_(b, A, h)),
        "apply_q": ({}, lambda b, A, al: D.apply_q_(b, A, h)),
        "backsolve bs_wave=1": ({"bs_wave": 1}, lambda b, A, al: D.backsolve_(b, A, al, h)),
        "backsolve bs_wave=0": ({"bs_wave": 0}, lambda b, A, al: D.backsolve_(b, A, al, h)),
        "solve": ({}, lambda b, A, al: D.solve_householder_(b, A, al, h)),
    }


def rhs_layouts(m):
    """(nrhs, ldb, misaligned): a vector at offsets 0 and 8 B, and blocks of 3 and 65 with ldb in {m, m+1, m+2} x both bases."""
    out = [(1, m, False), (1, m, True)]
    for nrhs in (3, 65):
        out += [(nrhs, m + e, mis) for e in (0, 1, 2) for mis in (False, True)]
    return out


@pytest.mark.parametrize("m,n", SHAPES, ids=[f"{m}x{n}" for m, n in SHAPES])
def test_solves_are_bitwise_independent_of_the_layouts(D, h, m, n):
    H0 = D.to_colmajor(matrix(m + n, m, n), DEV)
    a0 = factor(D, h, H0, 0)
    ops = solve_ops(D, h)
    B0 = {k: matrix(7 + k, m, k) for k in (1, 3, 65)}
    ref = {}
    for op, (opts, fn) in ops.items():                     # L0 everywhere: A as factored, b plain (vector / ldb = m)
        with options(h, **opts):
            for k, B in B0.items():
                b = B[:, 0].clone() if k == 1 else D.to_colmajor(B, DEV)
                fn(b, H0, a0)
                ref[(op, k)] = b
    torch.cuda.synchronize()
    for name in ["L0"] + list(layouts(m)):
        if name == "L0":
            GA, A = None, H0
        else:
            GA = guarded_layout(name, m, n)
            GA.A.copy_(H0)
            A = GA.A
        for op, (opts, fn) in ops.items():
            with options(h, **opts):
                for k, ldb, mis in rhs_layouts(m):
                    Gb = placed(m, k, ldb, mis)
                    Gb.A.copy_(B0[k])
                    b = Gb.vec if k == 1 else Gb.A
                    fn(b, A, a0)
                    torch.cuda.synchronize()
                    where = f"{op}, {m}x{n}, A in {name}, nrhs {k}, ldb {ldb}, b {'8 B off' if mis else '16 B'}"
                    assert_bitwise(b, ref[(op, k)], where)
                    Gb.check("b: " + where)
        if GA is not None:
            assert_bitwise(GA.A, H0, f"A is read only; layout {name}")
            GA.check(f"A: solves on layout {name}")
    # the C-ABI with nrhs = 1 and ldb = m + 3: a single right-hand side never uses ldb (both sweeps of Q'b / Qb: the GEMV-shaped
    # one, and the block update with qt_vec = 0, which sums in another order; each against the same sweep on a plain vector)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for fn, op in (("dhqr_apply_qt_f64", "apply_qt qt_vec=1"), ("dhqr_apply_q_f64", "apply_q"), ("dhqr_solve_f64", "solve")):
        for qv in (1, 0):
            with options(h, qt_vec=qv):
                b = B0[1][:, 0].clone()
                ops[op][1](b, H0, a0)
                Gb = Guarded(m, 1, m + 3, 0, 1)
                Gb.A.copy_(B0[1])
                alpha = (C.c_void_p(a0.data_ptr()),) if fn == "dhqr_solve_f64" else ()
                D._lib.call(fn, h.raw, m, n, 0, n, C.c_void_p(H0.data_ptr()), m, *alpha, C.c_void_p(Gb.A.data_ptr()), m + 3, 1, st)
                torch.cuda.synchronize()
                assert_bitwise(Gb.vec, b, f"{fn} nrhs 1 ldb m+3 qt_vec {qv}")
                Gb.check(f"{fn} nrhs 1 ldb m+3 qt_vec {qv}")


# ---------------------------------------------------------------------------------------------------------------------
# form_q_f64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,n", SHAPES, ids=[f"{m}x{n}" for m, n in SHAPES])
def test_form_q_is_bitwise_independent_of_the_layouts(D, h, m, n):
    H0 = D.to_colmajor(matrix(m + n, m, n), DEV)
    factor(D, h, H0, 0)
    Hkeep = H0.clone()
    Q0 = D.form_q(H0, handle=h)
    torch.cuda.synchronize()
    assert_bitwise(H0, Hkeep, "form_q out of place leaves A alone")
    for name in layouts(m):
        GQ = guarded_layout(name, m, n)                    # Q in the layout, A in L0
        D.form_q(H0, out=GQ.A, handle=h)
        torch.cuda.synchronize()
        assert_bitwise(GQ.A, Q0, f"Q in {name}")
        GQ.check(f"Q in {name}")
        assert_bitwise(H0, Hkeep, f"A in L0 after Q in {name}")
        GA = guarded_layout(name, m, n)                    # A in the layout, Q in L0
        GA.A.copy_(H0)
        Q = D.form_q(GA.A, handle=h)
        torch.cuda.synchronize()
        assert_bitwise(Q, Q0, f"A in {name}")
        assert_bitwise(GA.A, H0, f"A in {name} is read only")
        GA.check(f"A in {name}")
        D.form_q(GA.A, out=GA.A, handle=h)                 # in place
        torch.cuda.synchronize()
        assert_bitwise(GA.A, Q0, f"in place in {name}")
        GA.check(f"in place in {name}")
    Hin = H0.clone()
    D.form_q(Hin, out=Hin, handle=h)
    torch.cuda.synchronize()
    assert_bitwise(Hin, Q0, "in place in L0")


# ---------------------------------------------------------------------------------------------------------------------
# ComplexF64
# ---------------------------------------------------------------------------------------------------------------------
C_SHAPES = [(1000, 300), (333, 129)]


def c_layouts(m):
    """(lda, row offset in complex elements); one guard column on each side"""
    return [(m + e, r0) for e in (0, 1, 2) for r0 in (0, 1, 2)]


@pytest.mark.parametrize("m,n", C_SHAPES, ids=[f"{m}x{n}" for m, n in C_SHAPES])
def test_complex_is_bitwise_independent_of_the_layout(D, h, m, n):
    cd = torch.complex128
    A0 = matrix(m + n, m, n, cd)
    b1, b3 = matrix(5, m, 1, cd), matrix(6, m, 3, cd)
    H0 = D.to_colmajor(A0, DEV)
    a0 = factor(D, h, H0, 0)
    ref = {}
    for k, B in ((1, b1), (3, b3)):
        for op in ("apply_qt", "backsolve", "solve"):
            b = B[:, 0].clone() if k == 1 else D.to_colmajor(B, DEV)
            if op == "apply_qt":
                D.apply_qt_(b, H0, h)
            elif op == "backsolve":
                D.backsolve_(b, H0, a0, h)
            else:
                D.solve_householder_(b, H0, a0, h)
            ref[(op, k)] = b
    Q0 = D.form_q(H0, handle=h)
    torch.cuda.synchronize()
    for lda, r0 in c_layouts(m):
        where = f"ComplexF64 {m}x{n}, lda m+{lda - m}, {r0} rows above"
        G, ga = Guarded(m, n, lda, r0, 1, cd), Guarded(n, 1, n, 1, 1, cd)
        G.A.copy_(A0)
        a = factor(D, h, G.A, 0, ga)
        assert_bitwise(G.A, H0, "H: " + where)
        assert_bitwise(a, a0, "alpha: " + where)
        G.check("qr: " + where)
        ga.check("alpha: " + where)
        for k, B in ((1, b1), (3, b3)):
            for op in ("apply_qt", "backsolve", "solve"):
                Gb = Guarded(m, k, lda, r0, 1, cd)
                Gb.A.copy_(B)
                b = Gb.vec if k == 1 else Gb.A
                if op == "apply_qt":
                    D.apply_qt_(b, G.A, h)
                elif op == "backsolve":
                    D.backsolve_(b, G.A, a, h)
                else:
                    D.solve_householder_(b, G.A, a, h)
                torch.cuda.synchronize()
                assert_bitwise(b, ref[(op, k)], f"{op} nrhs {k}: {where}")
                Gb.check(f"b of {op} nrhs {k}: {where}")
        assert_bitwise(G.A, H0, "A is read only in the solves: " + where)
        GQ = Guarded(m, n, lda, r0, 1, cd)
        D.form_q(H0, out=GQ.A, handle=h)
        torch.cuda.synchronize()
        assert_bitwise(GQ.A, Q0, "form_q out of place: " + where)
        GQ.check("form_q out of place: " + where)
        D.form_q(G.A, out=G.A, handle=h)
        torch.cuda.synchronize()
        assert_bitwise(G.A, Q0, "form_q in place: " + where)
        G.check("form_q in place: " + where)


def test_complex_entry_points_reject_8_byte_aligned_pointers(D, h):
    # A ComplexF64 pointer that is only 8 B aligned is legal C but the complex kernels move double2: every complex entry point
    # turns it down with -(1-based index of the argument) before anything is enqueued.  Every buffer has one spare element, so
    # the shifted pointers stay inside their allocations.
    lib = D._lib.load()
    cd = torch.complex128
    m, n = 96, 40
    bufs = {k: torch.randn(s + 1, dtype=cd, device=DEV) for k, s in (("A", m * n), ("alpha", n), ("b", m), ("Q", m * n), ("out", 1))}
    torch.cuda.synchronize()
    keep = {k: v.clone() for k, v in bufs.items()}
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    # entry point -> its pointer arguments as (buffer, code): the rest of the argument list is built around them
    cases = {
        "dhqr_qr_c64": (("A", -6), ("alpha", -8)),
        "dhqr_apply_qt_c64": (("A", -6), ("b", -8)),
        "dhqr_backsolve_c64": (("A", -6), ("alpha", -8), ("b", -9)),
        "dhqr_solve_c64": (("A", -6), ("alpha", -8), ("b", -9)),
        "dhqr_form_q_c64": (("A", -4), ("Q", -6)),
        "dhqr_partialdot_c64": (("A", -2), ("b", -3), ("out", -6)),
    }

    def args(fn, bad):
        p = {k: C.c_void_p(v.data_ptr() + (8 if k == bad else 0)) for k, v in bufs.items()}
        if fn == "dhqr_qr_c64":
            return h.raw, m, n, 0, n, p["A"], m, p["alpha"], st
        if fn == "dhqr_apply_qt_c64":
            return h.raw, m, n, 0, n, p["A"], m, p["b"], m, 1, st
        if fn in ("dhqr_backsolve_c64", "dhqr_solve_c64"):
            return h.raw, m, n, 0, n, p["A"], m, p["alpha"], p["b"], m, 1, st
        if fn == "dhqr_form_q_c64":
            return h.raw, m, n, p["A"], m, p["Q"], m, st
        return h.raw, p["A"], p["b"], 0, m, p["out"], st

    for fn, ptrs in cases.items():
        for bad, code in ptrs:
            before = h.launch_count()
            rc = getattr(lib, fn)(*args(fn, bad))
            assert rc == code, f"{fn} with {bad} 8 B off a 16 B boundary returned {rc}, expected {code}: {lib.dhqr_last_error().decode()}"
            assert "16-byte" in lib.dhqr_last_error().decode(), fn
            assert h.launch_count() == before, f"{fn} with a misaligned {bad} launched a kernel"
            torch.cuda.synchronize()
            for k, v in bufs.items():
                assert_bitwise(v, keep[k], f"{fn} with a misaligned {bad} changed {k}")


# ---------------------------------------------------------------------------------------------------------------------
# host entry
# ---------------------------------------------------------------------------------------------------------------------
class HostGuarded:
    """Guarded operand in host memory: pinned (a torch pinned buffer seen through numpy) or pageable (numpy)."""

    def __init__(self, m, n, ld, g=1, pinned=True):
        size = (n + 2 * g) * ld
        self.pinned = torch.empty(size, dtype=torch.float64).pin_memory() if pinned else None
        self.buf = self.pinned.numpy() if pinned else np.empty(size)
        self.words = self.buf.view(np.int64)
        self.words[:] = SENTINEL
        self.A = np.lib.stride_tricks.as_strided(self.buf[g * ld:], shape=(m, n), strides=(8, 8 * ld))
        self.outside = np.ones(size, dtype=bool)
        np.lib.stride_tricks.as_strided(self.outside[g * ld:], shape=(m, n), strides=(1, ld))[:] = False
        self.ptr = C.c_void_p(self.A.ctypes.data)

    def check(self, where):
        bad = (self.words != SENTINEL) & self.outside
        assert not bad.any(), f"{int(bad.sum())} host words outside the operand changed, the first at {int(np.flatnonzero(bad)[0])}; {where}"


def host_qr(D, h, A0, ld, nb, pinned):
    m, n = A0.shape
    HA, Ha = HostGuarded(m, n, ld, 1, pinned), HostGuarded(n, 1, n, 1, pinned)
    HA.A[:] = A0
    D._lib.call("dhqr_qr_host_f64", h.raw, m, n, HA.ptr, ld, Ha.ptr, nb)
    return HA, Ha


@pytest.mark.parametrize("nb", [0, 1])
def test_host_entry_is_bitwise_independent_of_the_host_layout(D, h, nb):
    m, n = HOST_SHAPE
    A0 = matrix(21, m, n).cpu().numpy()
    b = matrix(22, m, 1).cpu().numpy()[:, 0].copy()
    for chunk in (128, 512):
        with options(h, host_chunk=chunk):
            ref = None
            for ld, pinned in ((m, True), (m + 1, True), (m + 5, True), (m + 1, False)):
                where = f"nb {nb}, host_chunk {chunk}, host lda m+{ld - m}, {'pinned' if pinned else 'pageable'}"
                HA, Ha = host_qr(D, h, A0, ld, nb, pinned)
                HA.check("A: " + where)
                Ha.check("alpha: " + where)
                got = (np.array(HA.A), np.array(Ha.A[:, 0]))
                if ref is None:
                    ref = got
                    continue
                for x, y, what in ((got[0], ref[0], "H"), (got[1], ref[1], "alpha")):
                    ne = x.view(np.int64) != y.view(np.int64)
                    assert not ne.any(), f"{what}: {int(ne.sum())} entries differ in their bits from host lda m, pinned; {where}"
    # dhqr_ldiv_host_f64 from a factorisation with host lda > m, a guard after x; b is read only
    H, a = ref
    xs = []
    for ld in (m, m + 5):
        HA, Ha = HostGuarded(m, n, ld), HostGuarded(n, 1, n)
        HA.A[:] = H
        Ha.A[:, 0] = a
        Hb, Hx = HostGuarded(m, 1, m), HostGuarded(n, 1, n)
        Hb.A[:, 0] = b
        D._lib.call("dhqr_ldiv_host_f64", h.raw, m, n, HA.ptr, ld, Ha.ptr, Hb.ptr, Hx.ptr)
        for G, what in ((HA, "A"), (Ha, "alpha"), (Hb, "b"), (Hx, "x")):
            G.check(f"ldiv_host {what}, host lda m+{ld - m}")
        assert np.array_equal(HA.A.view(np.int64), H.view(np.int64)) and np.array_equal(Hb.A[:, 0].view(np.int64), b.view(np.int64))
        xs.append(np.array(Hx.A[:, 0]))
    assert np.isfinite(xs[0]).all()
    assert np.array_equal(xs[0].view(np.int64), xs[1].view(np.int64)), "ldiv_host x depends on the host lda"


# ---------------------------------------------------------------------------------------------------------------------
# primitives
# ---------------------------------------------------------------------------------------------------------------------
def test_fill_uniform_is_bitwise_independent_of_the_layout(D, h):
    m, n = 1537, 40
    A0 = D.colmajor_empty(m, n, DEV)
    D.fill_uniform_(A0, 9, 5, 3, handle=h)
    for name in list(layouts(m)) + ["ld m, 8 B off"]:
        G = placed(m, n, m, True) if name == "ld m, 8 B off" else guarded_layout(name, m, n)
        D.fill_uniform_(G.A, 9, 5, 3, handle=h)
        torch.cuda.synchronize()
        assert_bitwise(G.A, A0, f"fill_uniform in {name}")
        G.check(f"fill_uniform in {name}")


@pytest.mark.parametrize("dtype", [torch.float64, torch.complex128], ids=["f64", "c64"])
def test_partialdot_reads_only_its_range(D, h, dtype):
    N = 5000
    for i0, i1 in ((0, N), (1, N - 1), (37, 4001), (2500, 2501), (100, 100)):
        data_a, data_b = matrix(i0 + 1, i1 - i0, 1, dtype)[:, 0], matrix(i1 + 2, i1 - i0, 1, dtype)[:, 0]
        ga, gb = Guarded(N, 1, N, 0, 1, dtype), Guarded(N, 1, N, 0, 1, dtype)
        pa, pb = matrix(3, N, 1, dtype)[:, 0], matrix(4, N, 1, dtype)[:, 0]
        for G, P, d in ((ga, pa, data_a), (gb, pb, data_b)):
            G.vec[i0:i1] = d
            P[i0:i1] = d
        keep = (ga.words.clone(), gb.words.clone())
        got = D.partialdot(ga.vec, gb.vec, range(i0, i1), h)
        plain = D.partialdot(pa, pb, range(i0, i1), h)
        where = f"partialdot {dtype} [{i0}, {i1})"
        assert np.isfinite(got), where
        assert np.array_equal(np.array([got]).view(np.int64), np.array([plain]).view(np.int64)), f"{got!r} != {plain!r}; {where}"
        assert torch.equal(ga.words, keep[0]) and torch.equal(gb.words, keep[1]), where
