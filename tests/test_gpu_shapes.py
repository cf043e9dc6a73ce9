"""The extended-precision rule of tests/ext_rule.py at the shape edges (run with -m gpu on an H100).

test_gpu_ext.py holds every path to err_gpu <= C_REL max(err_fp64_oracle, FLOOR) on hard families, at shapes whose last outer
panel still has a thousand rows below it.  This module puts the same rule on the bottom-right corner of near-square matrices,
where the tail code runs: partial 64-row chunks of the wide chain, the last 32-row strip, windows narrower than a tile,
reflectors of length 1; and on right-hand-side widths either side of the 64-column tiles, complex shapes at the 64-column
panel boundary, the host entry with a short last chunk, and a handle's history.

Each extended / fp64 reference is computed once per (family, shape) and shared by every path at that shape.  A table of the
worst ratio per (shape, path) x family is written to build/test_gpu_shapes_ratios.md.
"""
import numpy as np
import pytest
import torch

import matrix_families as F
from ext_rule import C_REL, Ref, Table, digest, factor_checks, nrm, options, run_qr

pytestmark = pytest.mark.gpu

# shape -> (m, n); the boundary each one hits.  The blocked driver works in 128-column outer panels; a full panel whose window
# (rows from its pivot row down) has >= 128 rows goes through the wide chain (CholeskyQR2 + reconstruction, k_vpk_rmul over
# 64-row chunks of a window rounded up to 128 rows: chunks 0-1 are the top block, the final pass covers chunks 2 .. nq - 1);
# any other panel through the narrow chain (k_panel over 32-column inner panels).
SHAPES = {
    "1024x1024": (1024, 1024),   # last wide panel on a 128-row window: nq = 2, the final k_vpk_rmul pass is empty
    "1025x1024": (1025, 1024),   # last wide window 129 rows: chunk 2 holds one live row, chunk 3 is dead
    "1087x1024": (1087, 1024),   # 191 rows: chunk 2 full, chunk 3 all dead but one row short of a chunk
    "1088x1024": (1088, 1024),   # 192 rows: chunk 2 full, chunk 3 dead
    "1151x1024": (1151, 1024),   # 255 rows: chunk 3 one row short
    "1000x1000": (1000, 1000),   # last outer panel 104 columns (narrow), last inner panel 8 x 8, back-solve strip of 8 rows
    "1001x1000": (1001, 1000),   # k_panel windows of 9 rows ...
    "1031x1000": (1031, 1000),   # ... 39 ...
    "1032x1000": (1032, 1000),   # ... 40 ...
    "1033x1000": (1033, 1000),   # ... and 41 rows at the last inner panel
    "993x993": (993, 993),       # one-row last reflector (H = -1); n = 31 * 32 + 1: a one-row last back-solve strip
    "1023x1023": (1023, 1023),   # n = 31 (mod 32), m = 63 (mod 64): 31 x 31 last inner panel
    "1153x1025": (1153, 1025),   # a one-column outer panel (129-row window) after 8 full wide ones (last wide window 257 rows)
    "128x128": (128, 128),       # the whole matrix one wide panel on a 128-row window, one split-K chunk pair
    "129x128": (129, 128),       # one wide panel, 129-row window
    "160x160": (160, 160),       # one wide panel + a 32-column narrow panel on a 32-row window
    "65x33": (65, 33),           # two inner panels, the second one column on 33 rows; single-chunk split-K
    "33x32": (33, 32),           # one inner panel with one row below it
    "2x2": (2, 2),
    "1x1": (1, 1),
}
# k_unblocked_wave keeps its column in registers, UW_MAXI = 32 rows per thread at 256 threads; square matrices on either side
# of a 256-row register tile and the last pivot handed to thread 1 of a 2-row tail (nb = 1 only)
NB1_SHAPES = {"255x255": (255, 255), "256x256": (256, 256), "257x257": (257, 257)}

# path -> (nb, extra rows of lda, options)
PATHS = {
    "default": (0, 0, {}),                       # wide chain + look-ahead
    "wide_panel0": (0, 0, {"wide_panel": 0}),    # narrow chain only
    "nb64": (64, 0, {}),                         # 64-column outer panels (narrow chain)
    "lookahead0_lda+1": (0, 1, {"lookahead": 0}),   # serial schedule with the wide chain, odd leading dimension
    "nb1": (1, 0, {}),                           # one reflector per step (k_unblocked_wave up to 8192 rows)
}
WIDE_PATHS = ("default", "lookahead0_lda+1")
FAMILIES = ("uniform", "normal", "graded12", "colscale", "kahan")
# well-conditioned: every full panel must be accepted by the wide chain, the last one included.  At 1024 x 1024 .. 1151 x 1024
# that is the last panel on a 128 .. 255-row window, so these rows are known to have run through the wide chain's tail.
ACCEPTED = ("uniform", "normal")

ALL_SHAPES = dict(SHAPES, **NB1_SHAPES)
# the Kahan matrix needs (1 + c)^(n - 1) = 1e8 with c < 1, i.e. n >= 28; below that (2 x 2, 1 x 1) it is left out
CASES = [(s, p, f) for s in ALL_SHAPES for f in FAMILIES for p in (PATHS if s in SHAPES else ("nb1",))
         if not (f == "kahan" and ALL_SHAPES[s][1] < 28)]

TABLE = Table("test_gpu_shapes_ratios.md")
# kappa = 1e12 on a small matrix: the fp64 oracle's error is one sample of a spread set by the summation order, not a bound.
# Measured on an H100 80GB HBM3 SXM at 700 W: at 160 x 160 the V error of every blocked path is 2.2e-5, 9.5 x the oracle's
# 2.3e-6 (nb = 64: 6.9 x, nb = 1: 0.8 x), while the oracle's own recurrences summed in numpy's order land at 4.5e-6.  This
# cell gets 16 instead of C_REL.
C_REL_SUMMATION = {("160x160", "graded12"): 16}


def c_rel(shape, family):
    return C_REL_SUMMATION.get((shape, family), C_REL)


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    TABLE.write()


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="module")
def refs(oracle, coracle):
    # the cases of one shape run back to back: every other shape is dropped once the next one is asked for
    cache = {}

    def get(family, m, n, cplx=False, nrhs=1):
        key = (family, m, n, cplx, nrhs)
        if key not in cache:
            for old in [c for c in cache if c[1:3] != (m, n)]:
                del cache[old]
            cache[key] = Ref(coracle, oracle, family, m, n, cplx=cplx, nrhs=nrhs)
        return cache[key]
    return get


def check_regime(label, path, ref, delta, note):
    where = f"{label}, family {ref.family}; {note}"
    if path not in WIDE_PATHS:
        assert delta["wide_panels"] == 0 and delta["wide_redone"] == 0, f"the wide chain ran on a narrow path; {where}"
        return
    TABLE.counts[(label, ref.family)] = (delta["wide_panels"], delta["wide_redone"])
    if ref.family in ACCEPTED:
        assert delta["wide_panels"] == ref.n // 128 and delta["wide_redone"] == 0, \
            f"every full panel, the last one included, should go through the wide chain; {where}"


def check_solves(D, label, ref, dA, st, c_rel=C_REL):
    """Q'b through the GEMV-shaped sweep (qt_vec = 1) and the block update (0), Qb, and x by the wavefront back-substitution
    (bs_wave = 1) and by k_backsolve_step blocks (0): one right-hand side, against the extended reference."""
    h = st.handle
    b = torch.from_numpy(ref.b[:, 0].copy()).cuda()
    for qv in (1, 0):
        with options(h, qt_vec=qv):
            qtb = D.apply_qt_(b.clone(), dA).cpu().numpy()
        g, e = ref.solve_errors("qtb", qtb, 0)
        TABLE.check(label, ref, {"qtb": g}, {"qtb": e}, note=f"apply_qt qt_vec={qv}", c_rel=c_rel)
    g, e = ref.solve_errors("qb", D.apply_q_(b.clone(), dA).cpu().numpy(), 0)
    TABLE.check(label, ref, {"qb": g}, {"qb": e}, note="apply_q", c_rel=c_rel)
    for bw in (1, 0):
        with options(h, bs_wave=bw):
            x = D.ldiv(st, b).cpu().numpy()
        g, e = ref.solve_errors("x", x, 0)
        TABLE.check(label, ref, {"x": g}, {"x": e}, note=f"ldiv bs_wave={bw}", c_rel=c_rel)


@pytest.mark.parametrize("shape,path,family", CASES, ids=[f"{s}-{p}-{f}" for s, p, f in CASES])
def test_shape(D, refs, shape, path, family):
    m, n = ALL_SHAPES[shape]
    nb, extra, opts = PATHS[path]
    ref = refs(family, m, n)
    label = f"{shape} {path}"
    dA, st, note, delta = run_qr(D, ref.A, nb, extra, **opts)
    check_regime(label, path, ref, delta, note)
    H, alpha = dA.cpu().numpy(), st.α.cpu().numpy()
    gpu, absolute = factor_checks(label, ref, H, alpha, note)
    TABLE.check(label, ref, gpu, ref.e64, absolute, note, c_rel(shape, family))
    if ref.solve:
        check_solves(D, label, ref, dA, st, c_rel(shape, family))


# ---------------------------------------------------------------------------------------------------------------------
# right-hand-side widths: apply_block_reflector tiles nrhs columns as 64-column k_gemm_vta / k_gemm_cvy tiles and YCOLS groups
# in k_ymake; the workspace is sized by max(n, nrhs), so nrhs > n (200 > 37) is a case of its own
# ---------------------------------------------------------------------------------------------------------------------
WIDTHS = (1, 2, 63, 64, 65, 129, 200)       # nrhs = 1 with qt_vec = 0: the block update, not the GEMV-shaped sweep


@pytest.fixture(scope="module")
def wide_refs(oracle, coracle):
    cache = {}

    def get(family, m, n, cplx=False):
        key = (family, m, n, cplx)
        if key not in cache:
            cache.clear()
            cache[key] = Ref(coracle, oracle, family, m, n, cplx=cplx, nrhs=65 if cplx else max(WIDTHS))
        return cache[key]
    return get


def check_block(label, ref, results, note):
    """Each metric over a block of right-hand sides: the block's worst column against the fp64 oracle's worst column.  At
    kappa = 1e12 the oracle's error on one column is a single sample spread over three decades (x at 300 x 37: 4.9e-7 ... 2.3e-4
    over 200 columns; LAPACK lands at 8e-5 on a column where the oracle has 9e-6), so a column-by-column ratio would measure
    luck.  On well-conditioned input every column sits near the same error, and a wrong column tile raises the block's worst."""
    gpu, e64 = {}, {}
    for key, got in results.items():
        errs = [ref.solve_errors(key, got[:, r], r) for r in range(got.shape[1])]
        gpu[key], e64[key] = max(g for g, _ in errs), max(e for _, e in errs)
    TABLE.check(label, ref, gpu, e64, note=note)


def rhs_block(D, B0, ldb):
    B = D.colmajor_empty(B0.shape[0], B0.shape[1], "cuda:0", lda=ldb, dtype=torch.from_numpy(B0[:1, :1]).dtype)
    B.copy_(torch.from_numpy(B0))
    return B


@pytest.mark.parametrize("nrhs", WIDTHS)
@pytest.mark.parametrize("family", ("normal", "graded12"))
@pytest.mark.parametrize("mn", [(1000, 300), (300, 37)], ids=["1000x300", "300x37"])
def test_rhs_widths(D, wide_refs, mn, family, nrhs):
    m, n = mn
    ref = wide_refs(family, m, n)
    dA, st, note, _ = run_qr(D, ref.A)
    B0 = np.asfortranarray(ref.b[:, :nrhs])
    h = D.default_handle(0)
    with options(h, qt_vec=0 if nrhs == 1 else h.get_option("qt_vec")):
        Q = D.apply_qt_(rhs_block(D, B0, m + 1), dA).cpu().numpy()
        P = D.apply_q_(rhs_block(D, B0, m + 1), dA).cpu().numpy()
        X = D.solve_householder_(rhs_block(D, B0, m + 1), dA, st.α).cpu().numpy()
    check_block(f"{m}x{n} nrhs={nrhs} ldb=m+1", ref, {"qtb": Q, "qb": P, "x": X}, note)


@pytest.mark.parametrize("nrhs", (1, 2, 65))
@pytest.mark.parametrize("family", F.COMPLEX_FAMILIES)
def test_complex_rhs_widths(D, wide_refs, family, nrhs):
    m, n = 300, 37
    ref = wide_refs(family, m, n, cplx=True)
    dA, st, note, _ = run_qr(D, ref.A)
    B0 = np.asfortranarray(ref.b[:, :nrhs])
    Q = D.apply_qt_(rhs_block(D, B0, m + 1), dA).cpu().numpy()
    X = D.ldiv(st, torch.from_numpy(B0).cuda()).cpu().numpy()
    check_block(f"complex {m}x{n} nrhs={nrhs}", ref, {"qtb": Q, "x": X}, note)


# ---------------------------------------------------------------------------------------------------------------------
# complex: dhqr_qr_c64 factors 64-column panels (CPW) of the 2m-row real view
# ---------------------------------------------------------------------------------------------------------------------
COMPLEX_SHAPES = {
    "64x64": (64, 64, 0),        # exactly one CPW panel
    "65x64": (65, 64, 0),        # one panel, one row below it
    "128x128": (128, 128, 0),    # two panels; real view 256 rows: two full 128-row chunks
    "129x65": (129, 65, 0),      # a one-column second panel; real view 258 rows
    "127x127_lda+1": (127, 127, 1),   # odd lda, one-column-short second panel
    "1000x1000": (1000, 1000, 0),     # last panel 40 columns on 40 rows
    "1x1": (1, 1, 0),            # k_house1_c on one element
}


@pytest.mark.parametrize("family", F.COMPLEX_FAMILIES)
@pytest.mark.parametrize("shape", list(COMPLEX_SHAPES))
def test_complex_shape(D, refs, shape, family):
    m, n, extra = COMPLEX_SHAPES[shape]
    ref = refs(family, m, n, cplx=True, nrhs=None)
    dA, st, note, _ = run_qr(D, ref.A, 0, extra)
    H, alpha = dA.cpu().numpy(), st.α.cpu().numpy()
    label = f"complex {shape}"
    gpu, absolute = factor_checks(label, ref, H, alpha, note)
    b = torch.from_numpy(ref.b.copy()).cuda()
    gpu["qtb"] = nrm(D.apply_qt_(b.clone(), dA).cpu().numpy() - ref.qtb_e) / nrm(ref.b)
    gpu["x"] = nrm(D.ldiv(st, b).cpu().numpy() - ref.x_e) / nrm(ref.x_e)
    e64 = dict(ref.e64, qtb=nrm(ref.qtb64 - ref.qtb_e) / nrm(ref.b), x=nrm(ref.x64 - ref.x_e) / nrm(ref.x_e))
    TABLE.check(label, ref, gpu, e64, absolute, note)


# ---------------------------------------------------------------------------------------------------------------------
# host entry: 128-column upload chunks; the last one joins with a short window, so its catch-up runs on few rows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ("normal", "graded8"))
@pytest.mark.parametrize("mn", [(1152, 1152), (1153, 1024)], ids=["1152x1152", "1153x1024"])
def test_host_entry_corner(D, refs, mn, family):
    m, n = mn
    ref = refs(family, m, n)
    h = D.default_handle(0)
    A = ref.A.copy(order="F")
    with options(h, host_chunk=128):
        st = D.qr_(A)
    label = f"host {m}x{n} host_chunk=128"
    gpu, absolute = factor_checks(label, ref, A, st.α, "")
    gpu["x"], e_x = ref.solve_errors("x", D.ldiv(st, ref.b[:, 0].copy()), 0)
    TABLE.check(label, ref, gpu, dict(ref.e64, x=e_x), absolute)


# ---------------------------------------------------------------------------------------------------------------------
# handle history: the workspace of a handle only grows, and split counts, launch tags (bs_epoch, qt_ticket, the panel and
# wave epochs) and the wide chain's control block are per handle.  None of it may change the arithmetic.
# ---------------------------------------------------------------------------------------------------------------------
HISTORY = [(1024, 1024, 0), (1000, 1000, 0), (300, 37, 0), (1024, 1024, 1), (1000, 1000, 1), (300, 37, 1)]


def test_handle_history_is_bitwise_invisible(D):
    def run(h, m, n, nb):
        A0, b = F.make("normal", m, n), torch.from_numpy(F.rhs(m, 1)).cuda()
        dA, st, _, _ = run_qr(D, A0, nb, handle=h)
        qtb = D.apply_qt_(b.clone(), dA, handle=h)
        x = D.ldiv(st, b)
        torch.cuda.synchronize()
        return {"H": dA.cpu().numpy(), "alpha": st.α.cpu().numpy(), "Q'b": qtb.cpu().numpy(), "x": x.cpu().numpy()}

    fresh = D.Handle(0)
    try:
        first = {s: {k: digest(v) for k, v in run(fresh, *s).items()} for s in HISTORY}
    finally:
        fresh.close()
    run_qr(D, F.make("normal", 8192, 1024))            # the default handle, just after a larger factorisation
    for s in HISTORY:
        again = {k: digest(v) for k, v in run(D.default_handle(0), *s).items()}
        differ = [k for k in first[s] if first[s][k] != again[k]]
        assert not differ, f"{s[0]}x{s[1]} nb={s[2]}: {differ} differ between a fresh handle and one that factored 8192 x 1024"
