"""Every code path of the factorisation against the extended-precision reference, on inputs where kernels go wrong (run with
-m gpu on an H100).

The reference is oracle/dhqr_oracle.c's loop in long double (COracle.qr_ext): the reference's recurrences with a forward error
of about kappa * 1e-19.  The fp64 oracle runs the same loop in double, so its error against the extended reference on the
same input is what the reference algorithm in the reference's precision achieves.  The library is held to that:

    err_gpu <= C_REL * max(err_fp64_oracle, FLOOR)        for each metric below, on every family and path

Metrics (all against the extended reference; tests/matrix_families.py has the inputs):
    V     max |dH| over the lower trapezoid (the reflectors, entries O(1) since |v|^2 = 2)
    R     max |dR_ij| / ||A[:, j]|| over the strict upper triangle and alpha (column-relative: R spans 10^+-120 in colscale)
    qtb   ||d(Q'b)|| / ||b||          qb  ||d(Qb)|| / ||b||          x   ||dx|| / ||x||
FLOOR = 16 eps for V and R, 16 eps sqrt(m) for the solve metrics.  Two absolute bounds on every family inside the reference's
range:
    bwd   max_j ||(QR - A)[:, j]|| / ||A[:, j]|| < 1e-13
    orth  max_j | ||v_j||^2 - 2 | < 1e-13
Where a variant runs the same floating-point operations in the same order as another path, the two must agree bit for bit.

A table of err_gpu / max(err_fp64_oracle, FLOOR) per path x family is written to build/test_gpu_ext_ratios.md.  The rule, its
constants and the references live in tests/ext_rule.py, shared with test_gpu_shapes.py.
"""
import numpy as np
import pytest
import torch

import matrix_families as F
from ext_rule import COUNTERS, RHS, Ref, Table, counters, digest, factor_checks, nrm, options, run_qr

pytestmark = pytest.mark.gpu

# path -> (m, n, nb, extra rows of lda, options, path whose output it must equal bit for bit)
PATHS = {
    # blocked, default: 128-column wide chain + look-ahead
    "default": (2048, 1024, 0, 0, {}, None),
    # narrow (32-column) chain
    "wide_panel0": (2048, 1024, 0, 0, {"wide_panel": 0}, None),
    "nb32": (2048, 1024, 32, 0, {}, None),
    "nb64": (2048, 1024, 64, 0, {}, None),
    "nb96": (2048, 1024, 96, 0, {}, None),
    "panel_fast0": (2048, 1024, 0, 0, {"wide_panel": 0, "panel_fast": 0}, None),
    # serial schedules.  profile and sync both take the serial driver with the wide chain's side kernels on the main stream:
    # the same kernels, splits and order as lookahead = 0 (whose side stream only changes when they run)
    "lookahead0": (2048, 1024, 0, 0, {"lookahead": 0}, None),
    "profile1": (2048, 1024, 0, 0, {"profile": 1}, "lookahead0"),
    "sync1": (2048, 1024, 0, 0, {"sync": 1}, "lookahead0"),
    # cvy_persist = 0 launches k_gemm_cvy_p with one tile per CTA: the same tile code as the default walk
    "cvy_persist0": (2048, 1024, 0, 0, {"cvy_persist": 0}, "default"),
    # odd lda, a row count that is not a multiple of anything
    "lda+3": (4099, 640, 0, 3, {}, None),
    # nb = 1: persistent k_unblocked_wave (m <= 8192); fused k_house1 + k_apply1_tma chain (m <= 8531: its tile is sized by
    # (m + 2) & ~1 rows; odd lda at 8193 and 8531); above that one launch pair per column, k_apply1_tma while the tile of
    # (len + lead + 1) & ~1 rows fits 200 KiB: the whole of m = 8532, and k_apply1_direct for the first steps from m = 8533 on
    # (steps 0 and 1 at 8533, steps 0..469 at 9000; all of 32768 x 256 below)
    "nb1_m8192": (8192, 128, 1, 0, {}, None),
    "nb1_m8193": (8193, 128, 1, 0, {}, None),
    "nb1_m8531": (8531, 128, 1, 0, {}, None),
    "nb1_m8532": (8532, 128, 1, 0, {}, None),
    "nb1_m8533": (8533, 128, 1, 0, {}, None),
    "nb1_9000x600": (9000, 600, 1, 0, {}, None),
    "nb1_wave0": (4096, 512, 1, 0, {"unblocked_wave": 0}, None),
    "nb1_fuse0": (4096, 512, 1, 0, {"fuse_house": 0}, None),
    "nb1_lda+3": (4096, 512, 1, 3, {}, None),
}
BITWISE_TARGETS = {v[5] for v in PATHS.values() if v[5]}


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="session")
def refs(oracle, coracle):
    # the paths of one shape run back to back; 2048 x 1024 is shared by the solve and host-entry tests further down, every
    # other shape is dropped once the next one is asked for (a shape's set is up to ~0.4 GB of host memory)
    cache = {}
    keep = (2048, 1024)

    def get(family, m, n, k=None, cplx=False, solve=True):
        key = (family, m, n, k, cplx, solve)
        if key not in cache:
            for old in [c for c in cache if c[1:3] != (m, n) and c[1:3] != keep]:
                del cache[old]
            cache[key] = Ref(coracle, oracle, family, m, n, k, cplx, solve)
        return cache[key]
    return get


TABLE = Table("test_gpu_ext_ratios.md")
check = TABLE.check
COUNTS = TABLE.counts


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    TABLE.write()


ACCEPTED = ("uniform", "centered", "normal", "graded2")


def check_regime(path, ref, delta, note):
    """The wide chain's decisions: well-conditioned panels are all taken by it, a kappa = 1e12 spectrum at 4099 x 640 gets both
    verdicts, a zero column is refused and the factorisation restarts from that panel (the panels before it stay accepted)."""
    if path not in ("default", "lda+3"):
        return
    COUNTS[(path, ref.family)] = (delta["wide_panels"], delta["wide_redone"])
    where = f"path {path}, family {ref.family}, {ref.m}x{ref.n}; {note}"
    if ref.family in ACCEPTED:
        assert delta["wide_panels"] == ref.n // 128 and delta["wide_redone"] == 0, f"every panel should be accepted; {where}"
    if (path, ref.family) == ("lda+3", "graded12"):     # kappa = 1e12 at 4099 x 640 straddles the guard: both verdicts occur
        assert 1 <= delta["wide_redone"] < delta["wide_panels"], f"some panels accepted, some refused and redone; {where}"
    if ref.family == "zerocol_wide":
        assert delta["wide_redone"] >= 1 and delta["wide_panels"] >= F.zero_column(ref.family, ref.n) // 128, \
            f"the panel with the zero column should be refused and redone; {where}"


# ---------------------------------------------------------------------------------------------------------------------
# the path matrix
# ---------------------------------------------------------------------------------------------------------------------
_bitwise = {}


@pytest.mark.parametrize("family", F.FAMILIES)
@pytest.mark.parametrize("path", list(PATHS))
def test_path(D, refs, path, family):
    m, n, nb, extra, opts, same_as = PATHS[path]
    ref = refs(family, m, n)
    dA, st, note, delta = run_qr(D, ref.A, nb, extra, **opts)
    check_regime(path, ref, delta, note)
    H, alpha = dA.cpu().numpy(), st.α.cpu().numpy()
    gpu, absolute = factor_checks(path, ref, H, alpha, note)
    e64 = dict(ref.e64)
    if ref.solve:
        b = torch.from_numpy(ref.b[:, 0].copy()).cuda()
        qtb = D.apply_qt_(b.clone(), dA).cpu().numpy()
        x = D.ldiv(st, b).cpu().numpy()
        gpu["qtb"] = nrm(qtb - ref.qtb_e[:, 0]) / nrm(ref.b[:, 0])
        gpu["x"] = nrm(x - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])
        e64["qtb"] = nrm(ref.qtb64[:, 0] - ref.qtb_e[:, 0]) / nrm(ref.b[:, 0])
        e64["x"] = nrm(ref.x64[:, 0] - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])
    check(path, ref, gpu, e64, absolute, note)
    if path in BITWISE_TARGETS:
        _bitwise[(path, family)] = digest(H, alpha)
    if same_as:
        if (same_as, family) not in _bitwise:
            _, _, nb2, extra2, opts2, _ = PATHS[same_as]
            dB, st2, _, _ = run_qr(D, ref.A, nb2, extra2, **opts2)
            _bitwise[(same_as, family)] = digest(dB.cpu().numpy(), st2.α.cpu().numpy())
        assert digest(H, alpha) == _bitwise[(same_as, family)], \
            f"path {path} is not bitwise equal to path {same_as} on family {family}; {note}"


@pytest.mark.parametrize("family", [f for f in F.FAMILIES if f not in F.NAN_FAMILIES])
def test_solve_paths(D, refs, family):
    # Q'b with the GEMV-shaped sweep (qt_vec = 1) and the block update (0); Qb; back-substitution as one wavefront
    # (bs_wave = 1) and as k_backsolve_step blocks (0); three right-hand sides with ldb > m
    m, n = 2048, 1024
    ref = refs(family, m, n)
    dA, st, note, _ = run_qr(D, ref.A)
    h = D.default_handle(0)
    b = torch.from_numpy(ref.b[:, 0].copy()).cuda()
    nb_ = nrm(ref.b[:, 0])
    e_qtb64 = nrm(ref.qtb64[:, 0] - ref.qtb_e[:, 0]) / nb_
    e_x64 = nrm(ref.x64[:, 0] - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])
    for qv in (1, 0):
        with options(h, qt_vec=qv):
            qtb = D.apply_qt_(b.clone(), dA).cpu().numpy()
        check(f"apply_qt qt_vec={qv}", ref, {"qtb": nrm(qtb - ref.qtb_e[:, 0]) / nb_}, {"qtb": e_qtb64}, note=note)
    qb = D.apply_q_(b.clone(), dA).cpu().numpy()
    check("apply_q", ref, {"qb": nrm(qb - ref.qb_e[:, 0]) / nb_}, {"qb": nrm(ref.qb64[:, 0] - ref.qb_e[:, 0]) / nb_}, note=note)
    for bw in (1, 0):
        with options(h, bs_wave=bw):
            x = D.ldiv(st, b).cpu().numpy()
        check(f"ldiv bs_wave={bw}", ref, {"x": nrm(x - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])}, {"x": e_x64}, note=note)
    B = D.colmajor_empty(m, 3, "cuda:0", lda=m + 5)
    B.copy_(torch.from_numpy(ref.b[:, 1:]))
    Q = D.colmajor_empty(m, 3, "cuda:0", lda=m + 5)
    Q.copy_(B)
    D.apply_qt_(Q, dA)
    X = D.solve_householder_(B, dA, st.α).cpu().numpy()
    Q = Q.cpu().numpy()
    for r in range(1, RHS):
        nbr = nrm(ref.b[:, r])
        gpu = {"qtb": nrm(Q[:, r - 1] - ref.qtb_e[:, r]) / nbr, "x": nrm(X[:, r - 1] - ref.x_e[:, r]) / nrm(ref.x_e[:, r])}
        e64 = {"qtb": nrm(ref.qtb64[:, r] - ref.qtb_e[:, r]) / nbr, "x": nrm(ref.x64[:, r] - ref.x_e[:, r]) / nrm(ref.x_e[:, r])}
        check(f"nrhs=3 ldb=m+5 (rhs {r})", ref, gpu, e64, note=note)


@pytest.mark.parametrize("family", [f"graded{k}" for k in F.GRADED] + ["colscale"])
def test_host_entry(D, refs, family):
    # dhqr_qr_host_f64: upload in 128-column chunks that join the look-ahead schedule late, then dhqr_ldiv_host_f64
    m, n = 2048, 1024
    ref = refs(family, m, n)
    h = D.default_handle(0)
    A = ref.A.copy(order="F")
    with options(h, host_chunk=128):
        c0 = counters(h)
        st = D.qr_(A)
        c1 = counters(h)
    note = "counters " + ", ".join(f"{k} {c0[k]}->{c1[k]}" for k in COUNTERS)
    gpu, absolute = factor_checks("host host_chunk=128", ref, A, st.α, note)
    x = D.ldiv(st, ref.b[:, 0].copy())
    gpu["x"] = nrm(x - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])
    e64 = dict(ref.e64, x=nrm(ref.x64[:, 0] - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0]))
    check("host host_chunk=128", ref, gpu, e64, absolute, note)


@pytest.mark.parametrize("family", F.COMPLEX_FAMILIES)
def test_complex(D, refs, family):
    m, n = 1024, 384
    ref = refs(family, m, n, cplx=True)
    dA, st, note, _ = run_qr(D, ref.A)
    H, alpha = dA.cpu().numpy(), st.α.cpu().numpy()
    gpu, absolute = factor_checks("complex", ref, H, alpha, note)
    b = torch.from_numpy(ref.b.copy()).cuda()
    x = D.ldiv(st, b).cpu().numpy()
    gpu["qtb"] = nrm(D.apply_qt_(b.clone(), dA).cpu().numpy() - ref.qtb_e) / nrm(ref.b)
    gpu["x"] = nrm(x - ref.x_e) / nrm(ref.x_e)
    e64 = dict(ref.e64, qtb=nrm(ref.qtb64 - ref.qtb_e) / nrm(ref.b), x=nrm(ref.x64 - ref.x_e) / nrm(ref.x_e))
    check("complex", ref, gpu, e64, absolute, note)


LARGE_FAMILIES = ("uniform", "centered", "colscale", "rowscale")


@pytest.mark.parametrize("family", LARGE_FAMILIES)
@pytest.mark.parametrize("shape", [(32768, 4096, 0), (32768, 256, 1)], ids=["32768x4096", "32768x256-nb1"])
def test_large_shapes_leading_columns(D, oracle, coracle, shape, family):
    # BASELINE config 3 on the default path (its first 256 columns) and the nb = 1 direct-kernel path (all of H); not cached
    m, n, nb = shape
    ref = Ref(coracle, oracle, family, m, n, k=256, solve=False)
    dA, st, note, _ = run_qr(D, ref.A, nb)
    H, alpha = dA[:, :256].cpu().numpy(), st.α[:256].cpu().numpy()
    gpu, absolute = factor_checks(f"{m}x{n} nb={nb}", ref, H, alpha, note)
    check(f"{m}x{n} nb={nb}", ref, gpu, ref.e64, absolute, note)

