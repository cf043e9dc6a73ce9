"""Every Float64 path held to the extended-precision rule of tests/ext_rule.py at its height limits (run with -m gpu on an H100).

The kernels whose CTA geometry follows the row count are checked at the heights where that geometry changes:

A. qr_ at the panel-geometry heights.  k_panel, the 32-column chain's cooperative kernel, keeps a slab of up to 728 rows per CTA
   in shared memory on at most min(SMs, 160) CTAs, so lim = 728 S (S = min(SMs, 160)) is the tallest matrix the blocked paths
   take.  launch_panel starts from 64 CTAs under look-ahead, one per SM in the serial schedule, or the option panel_ctas, and
   doubles the CTA count while the slab does not fit.  The heights: lim, lim - 1, (S - 1) 728 + 1 (the last CTA holds one row),
   64 x 728 and one row more (either side of the first doubling under look-ahead).  n = 200: one 128-column panel for the wide
   chain, then a 72-column ragged panel that always goes through k_panel.  Every path factors, then Q'b (qt_vec 1 / 0), Qb, x
   (bs_wave 1 / 0), an nrhs = 3 block with ldb = m + 5 and the first 8 columns of form_q are held to the rule.  A zero column in
   panel 0 (a single panel) and in panel 1 (the second of a pair) makes the wide chain refuse it at full height and restart.
   One row past lim every blocked path returns -2 and leaves A alone; nb = 1 has no row limit.
B. The largest append: k = append_max_rows (the same slab rule in k_tp_panel), one row less, and a last CTA of one row; R', vtop
   and V2 against the stacked oracle, and Q~'[c; e] against the stacked oracle's Q'b.
C. Past a million rows: the one-vector Q'b sweep (k_qt_dot on at most 1024 CTAs of at most 1024 rows) takes m <= 2^20 and hands
   m = 2^20 + 1 to the block update.  nb = 1 and qrcp_ at both heights, with every solve that has a one-vector branch; the
   profiler shows which side of the switch ran.

Every height comes from the handle (sms, append_max_rows).  The ratio table goes to build/tall_ext.md.
"""
import os

import numpy as np
import pytest
import torch

import adjoint_oracle as AO
import cod_model as CM
import ext_rule as E
import matrix_families as F
from test_gpu_append import BLOCKED_ROW_GRADED, append, gpu_h, npy, stacked, start

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TABLE = E.Table("tall_ext.md")
MEMORY = {}                    # C: device memory a case took, (m, family) -> bytes

# launch_panel's rule (csrc/dhqr_api.cu), restated so that the heights below cannot drift from the cases they are meant to hit
IB, PANEL_MAXG, SLAB_BYTES = 32, 160, 184 * 1024
ROWS_MAX = ((SLAB_BYTES // (IB * 8)) - 4) & ~7          # 728 rows per CTA


def rup(x, a):
    return (x + a - 1) // a * a


def panel_geometry(mp, sms, lookahead, panel_ctas=0):
    """(rows per CTA, CTAs, rows in the last CTA, doublings) of k_panel on an mp-row window."""
    cap = min(sms, PANEL_MAXG)
    g = min(panel_ctas if panel_ctas > 0 else (64 if lookahead else sms), cap)
    rpc = rup(max(-(-mp // g), 64), 8)
    doublings = 0
    while IB * (rpc + 4) * 8 > SLAB_BYTES and g < cap:
        g = min(2 * g, cap)
        rpc = rup(max(-(-mp // g), 64), 8)
        doublings += 1
    G = -(-mp // rpc)
    return rpc, G, mp - (G - 1) * rpc, doublings


HEIGHTS = {
    "lim": lambda S: ROWS_MAX * S,
    "lim-1": lambda S: ROWS_MAX * S - 1,
    "last1": lambda S: (S - 1) * ROWS_MAX + 1,
    "la64": lambda S: 64 * ROWS_MAX,
    "la64+1": lambda S: 64 * ROWS_MAX + 1,
}
N = 200
# path -> (nb, options)
PATHS = {
    "default": (0, {}),
    "wide_panel0": (0, {"wide_panel": 0}),
    "panel_fast0": (0, {"wide_panel": 0, "panel_fast": 0}),
    "lookahead0": (0, {"lookahead": 0}),
    "nb64": (64, {}),
    "nb1": (1, {}),
}
PANEL_CTAS = (1, 7, 48, 160, 1000)
for _g in PANEL_CTAS:
    PATHS[f"panel_ctas{_g}"] = (0, {"wide_panel": 0, "panel_ctas": _g})
LIM_FAMILIES = ("normal", "graded6", "graded12", "colscale", "rowscale", "kahan", "tiny")
OTHER_FAMILIES = ("normal", "graded12")
CASES = [(hn, f, p) for hn in HEIGHTS for f in (LIM_FAMILIES if hn == "lim" else OTHER_FAMILIES)
         for p in PATHS if hn == "lim" or not p.startswith("panel_ctas")]
UNITS = 8                      # form_q's first columns, checked as Q e_j = Qb with b = e_j


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    return dhqr_b200


@pytest.fixture(scope="module")
def h(D):
    assert torch.cuda.is_available()
    hd = D.Handle(0)
    yield hd
    torch.cuda.synchronize()
    hd.close()


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    TABLE.write()
    if MEMORY:
        try:
            with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", TABLE.name), "a") as fh:
                fh.write("\ndevice memory per case past a million rows (fresh handle + operands):\n\n")
                fh.writelines(f"- {m} x 72 {f}: {b / 2**30:.2f} GiB\n" for (m, f), b in MEMORY.items())
        except OSError:
            pass


def S_of(h):
    return min(h.get_option("sms"), PANEL_MAXG)


def height(h, name):
    S = S_of(h)
    if name.startswith("la64") and S <= 64:
        pytest.skip(f"{S} panel CTAs: 64 x {ROWS_MAX} rows is past the row limit")
    return HEIGHTS[name](S)


_refs = {}


def ref_for(coracle, oracle, family, m, n, **kw):
    """One reference per (family, m, n), shared by the paths at that height; the cases run height by height and family by
    family, so only the current one is kept (a reference at the row limit holds ~0.5 GB of host memory)."""
    key = (family, m, n)
    if key not in _refs:
        _refs.clear()
        _refs[key] = E.Ref(coracle, oracle, family, m, n, **kw)
    return _refs[key]


def rhs_with_units(m):
    """Ref's default right-hand sides (column 0 alone, 1..3 as a block), then e_0 .. e_7 for form_q's columns."""
    return np.asfortranarray(np.hstack([F.rhs(m, E.RHS), np.eye(m, UNITS)]))


def check_solve(label, ref, key, got, r, note):
    g, e64 = ref.solve_errors(key, got, r)
    TABLE.check(label, ref, {key: g}, {key: e64}, note=f"{key} rhs {r}; {note}")


def check_solves(D, h, label, ref, dA, alpha, note):
    m = ref.m
    b0 = torch.from_numpy(ref.b[:, 0].copy()).to(DEV)
    for qv in (1, 0):
        with E.options(h, qt_vec=qv):
            got = D.apply_qt_(b0.clone(), dA, handle=h).cpu().numpy()
        check_solve(label, ref, "qtb", got, 0, f"qt_vec={qv}; {note}")
    check_solve(label, ref, "qb", D.apply_q_(b0.clone(), dA, handle=h).cpu().numpy(), 0, note)
    st = D.DistributedHouseholderQRStruct(dA, alpha, h)
    for bw in (1, 0):
        with E.options(h, bs_wave=bw):
            x = D.ldiv(st, b0).cpu().numpy()
        check_solve(label, ref, "x", x, 0, f"bs_wave={bw}; {note}")
    Q = D.colmajor_empty(m, 3, DEV, lda=m + 5)
    Q.copy_(torch.from_numpy(ref.b[:, 1:4]))
    X = D.colmajor_empty(m, 3, DEV, lda=m + 5)
    X.copy_(Q)
    D.apply_qt_(Q, dA, handle=h)
    X = D.solve_householder_(X, dA, alpha, handle=h).cpu().numpy()
    Q = Q.cpu().numpy()
    for r in range(1, 4):
        check_solve(label, ref, "qtb", Q[:, r - 1], r, f"nrhs=3 ldb=m+5; {note}")
        check_solve(label, ref, "x", X[:, r - 1], r, f"nrhs=3 ldb=m+5; {note}")
    Qf = D.form_q(dA, handle=h)[:, :UNITS].cpu().numpy()
    for j in range(UNITS):
        check_solve(label, ref, "qb", Qf[:, j], E.RHS + j, f"form_q column {j}; {note}")


def tries(widths):
    """k_panel launches that try the CholeskyQR2 fast path on outer panels of these widths: one per full 32-column inner panel
    (a narrower last one goes column by column untried); each advances panels_fast or panels_fallback by one."""
    return sum(w // IB for w in widths)


def panels(n, nb):
    w = nb or 128
    return [min(w, n - c) for c in range(0, n, w)]


def check_counters(path, nb, opts, n, delta, family, where):
    if nb == 1:
        assert all(v == 0 for v in delta.values()), f"nb = 1 runs no panel kernel; {where}"
        return
    narrow = panels(n, nb)
    tried = delta["panels_fast"] + delta["panels_fallback"]
    if nb == 0 and opts.get("wide_panel", 1):
        full = [w for w in narrow if w == 128]
        rest = [w for w in narrow if w != 128]
        assert delta["wide_panels"] == len(full), f"every full 128-column panel goes to the wide chain; {where}"
        assert delta["wide_redone"] <= 1, where          # only panel 0 can be refused
        if family == "normal":
            assert delta["wide_redone"] == 0, f"a well-conditioned panel was refused; {where}"
        # a refused panel is redone by the 32-column chain
        assert tried == tries(rest) + tries([128]) * delta["wide_redone"], where
        return
    assert delta["wide_panels"] == 0 and delta["wide_redone"] == 0, f"the wide chain ran with wide_panel = 0 or nb < 128; {where}"
    if opts.get("panel_fast", 1):
        assert tried == tries(narrow), where
    else:
        assert tried == 0, f"panel_fast = 0 never tries the fast path, so neither verdict counter moves; {where}"


# ---------------------------------------------------------------------------------------------------------------------
# A: qr_ at the panel-geometry heights
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hname", list(HEIGHTS))
def test_heights_hit_their_panel_geometry(h, hname):
    S = S_of(h)
    m = height(h, hname)
    assert ROWS_MAX == 728 and h.get_option("append_max_rows") == ROWS_MAX * S
    la, serial = panel_geometry(m, h.get_option("sms"), True), panel_geometry(m, h.get_option("sms"), False)
    where = f"{hname}: m = {m}, S = {S}, look-ahead (rows per CTA, CTAs, last, doublings) {la}, serial {serial}"
    if hname == "lim":
        for g in (la, serial) + tuple(panel_geometry(m, h.get_option("sms"), True, c) for c in PANEL_CTAS):
            assert g[:3] == (ROWS_MAX, S, ROWS_MAX), where
        assert panel_geometry(m + 1, h.get_option("sms"), False)[0] > ROWS_MAX, where   # one row more does not fit
    elif hname == "lim-1":
        assert la[:3] == serial[:3] == (ROWS_MAX, S, ROWS_MAX - 1), where
    elif hname == "last1":
        assert la[:3] == serial[:3] == (ROWS_MAX, S, 1), where
    elif hname == "la64":
        assert la == (ROWS_MAX, 64, ROWS_MAX, 0), where
    else:
        assert la[3] >= 1 and la[1] > 64 and la[0] < ROWS_MAX, where


@pytest.mark.parametrize("hname,family,path", CASES)
def test_path(D, h, coracle, oracle, hname, family, path):
    m = height(h, hname)
    nb, opts = PATHS[path]
    ref = ref_for(coracle, oracle, family, m, N, b=rhs_with_units(m))
    dA, st, note, delta = E.run_qr(D, ref.A, nb, handle=h, **opts)
    label = f"{path} m={hname}"
    where = f"path {path}, family {family}, {m}x{N}; {note}"
    check_counters(path, nb, opts, N, delta, family, where)
    if path == "default":
        TABLE.counts[(label, family)] = (delta["wide_panels"], delta["wide_redone"])
    gpu, absolute = E.factor_checks(label, ref, dA.cpu().numpy(), st.α.cpu().numpy(), note)
    TABLE.check(label, ref, gpu, ref.e64, absolute, note)
    if ref.solve:
        check_solves(D, h, label, ref, dA, st.α, note)


@pytest.mark.parametrize("n", (200, 256))
def test_restart_at_full_height(D, h, coracle, oracle, n):
    # n = 200: the zero column is in panel 0, a unit of its own; n = 256: in panel 1, the second of a pair, so the first panel's
    # reflectors are applied alone to the columns right of the pair before panel 1 is redone
    m = height(h, "lim")
    ref = ref_for(coracle, oracle, "zerocol_wide", m, n)
    assert F.zero_column("zerocol_wide", n) // 128 == (0 if n == 200 else 1)
    dA, st, note, delta = E.run_qr(D, ref.A, handle=h)
    label = f"restart n={n} m=lim"
    TABLE.counts[(label, ref.family)] = (delta["wide_panels"], delta["wide_redone"])
    assert delta["wide_redone"] >= 1 and delta["wide_panels"] == n // 128, f"the refused panel should be redone; {note}"
    gpu, absolute = E.factor_checks(label, ref, dA.cpu().numpy(), st.α.cpu().numpy(), note)   # incl. the oracle's NaN pattern
    TABLE.check(label, ref, gpu, ref.e64, absolute, note)


def test_row_limit(D, h, coracle, oracle):
    # one row past lim every blocked path is refused with -2 before it writes anything; nb = 1 has no row limit
    lim = height(h, "lim")
    A1 = F.make("normal", lim + 1, N)
    for path in ("default", "wide_panel0", "nb64", "lookahead0"):
        nb, opts = PATHS[path]
        dB = D.to_colmajor(A1, DEV)
        with E.options(h, **opts):
            with pytest.raises(D._lib.DhqrError) as e:
                D.qr_(dB, nb=nb, handle=h)
        assert e.value.code == -2, path
        torch.cuda.synchronize()
        assert np.array_equal(dB.cpu().numpy(), A1), f"path {path} wrote A before refusing it"
    del A1, dB
    m = lim + 1000
    ref = ref_for(coracle, oracle, "normal", m, N, solve=False)
    dA, st, note, delta = E.run_qr(D, ref.A, 1, handle=h)
    gpu, absolute = E.factor_checks("nb1 m=lim+1000", ref, dA.cpu().numpy(), st.α.cpu().numpy(), note)
    TABLE.check("nb1 m=lim+1000", ref, gpu, ref.e64, absolute, note)


# ---------------------------------------------------------------------------------------------------------------------
# B: the largest append
# ---------------------------------------------------------------------------------------------------------------------
APPEND_KS = {"cap": lambda cap, S: cap, "cap-1": lambda cap, S: cap - 1, "last1": lambda cap, S: (S - 1) * ROWS_MAX + 1,
             "700": lambda cap, S: 700}
APPEND_FAMILIES = ("normal", "graded6", "colscale", "kahan") + BLOCKED_ROW_GRADED


@pytest.mark.parametrize("family", APPEND_FAMILIES)
@pytest.mark.parametrize("kname", list(APPEND_KS))
def test_largest_append(D, h, coracle, oracle, kname, family):
    n, cap = 160, h.get_option("append_max_rows")
    k = APPEND_KS[kname](cap, S_of(h))
    st, B = start(D, h, family, n, k)
    alpha = st.α.cpu().numpy()
    Sk = stacked(npy(st.A), alpha, B)
    exempt = family in BLOCKED_ROW_GRADED
    b = None if exempt else F.rhs(n + k, 3, seed=9)
    ref = E.Ref(coracle, oracle, family, n + k, n, A=Sk, b=b, solve=not exempt)
    t = append(D, h, st, B)
    H = gpu_h(npy(st.A), st.α.cpu().numpy(), npy(t.B), t.vtop.cpu().numpy())
    label, note = f"append k={kname}", f"n={n} k={k}"
    gpu, absolute = E.factor_checks(label, ref, H, st.α.cpu().numpy(), note)
    if exempt:
        # test_gpu_append.py's exemption: on row-graded input the blocked structured algorithm is held to the absolute bounds
        for key, (val, tol) in absolute.items():
            assert val < tol, f"{key} = {val:.3e} >= {tol:.0e}; family {family}, {note}"
        return
    TABLE.check(label, ref, gpu, ref.e64, absolute, note)
    for nrhs in (1, 3):
        if nrhs == 1:
            c, e = (torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in (b[:n, 0], b[n:, 0]))
        else:
            c, e = D.to_colmajor(b[:n], DEV), D.to_colmajor(b[n:], DEV)
        t.apply_qt_(c, e)
        torch.cuda.synchronize()
        got = np.vstack([c.cpu().numpy().reshape(n, nrhs), e.cpu().numpy().reshape(k, nrhs)])
        for r in range(nrhs):
            check_solve(f"append Q~'[c;e] k={kname}", ref, "qtb", got[:, r], r, f"nrhs={nrhs}; {note}")


# ---------------------------------------------------------------------------------------------------------------------
# C: past a million rows
# ---------------------------------------------------------------------------------------------------------------------
MILLION = {"2^20": 1 << 20, "2^20+1": (1 << 20) + 1}
MILLION_N = 72
MILLION_FAMILIES = ("normal", "graded6")
NEED = 12 << 30                # device memory of a case, with headroom: 10.4 GiB measured on an H100 80GB HBM3 (written to the table)


def fresh_handle(D, m):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < NEED:
        pytest.skip(f"{m} x {MILLION_N} needs {NEED / 2**30:.0f} GiB of free device memory, {free / 2**30:.1f} GiB are free")
    return D.Handle(0), free


def record_memory(m, family, free0):
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    MEMORY[(m, family)] = max(used, MEMORY.get((m, family), 0))
    assert used <= NEED, f"{m} x {MILLION_N} took {used / 2**30:.2f} GiB of device memory, more than the {NEED / 2**30:.0f} GiB checked for"


def qt_dot_launches(h, call):
    """k_qt_dot launches of one call, from the profiler: the one-vector sweep ran iff there are any."""
    with E.options(h, profile=1):
        h.profile_reset()
        call()
        torch.cuda.synchronize()
        return h.profile().get("k_qt_dot", {"count": 0})["count"]


def check_switch(m, counts):
    """One k_qt_dot launch per sweep over the m rows (72 columns: one panel) where m <= 2^20, none past it.  solve_cod_ also
    applies Z, the factorisation of the 72-row R_r', with the one-vector sweep at any m."""
    for name, cnt in counts.items():
        want = (m <= 1 << 20) + (name == "solve_cod_")
        assert cnt == want, f"{name} at m = {m}: {cnt} k_qt_dot launches, not {want}; the one-vector sweep takes m <= 2^20 only"


@pytest.mark.parametrize("family", MILLION_FAMILIES)
@pytest.mark.parametrize("mname", list(MILLION))
def test_million_rows_qr(D, coracle, oracle, mname, family):
    m, n = MILLION[mname], MILLION_N
    hc, free0 = fresh_handle(D, m)
    try:
        ref = E.Ref(coracle, oracle, family, m, n, b=rhs_with_units(m), keep_h64=True)
        dA, st, note, _ = E.run_qr(D, ref.A, 1, handle=hc)
        label = f"nb1 m={mname}"
        gpu, absolute = E.factor_checks(label, ref, dA.cpu().numpy(), st.α.cpu().numpy(), note)
        TABLE.check(label, ref, gpu, ref.e64, absolute, note)
        b0 = torch.from_numpy(ref.b[:, 0].copy()).to(DEV)
        check_solve(label, ref, "qtb", D.apply_qt_(b0.clone(), dA, handle=hc).cpu().numpy(), 0, note)
        check_solve(label, ref, "qb", D.apply_q_(b0.clone(), dA, handle=hc).cpu().numpy(), 0, note)
        H = D.DistributedHouseholderQRStruct(dA, st.α, hc)
        check_solve(label, ref, "x", D.ldiv(H, b0).cpu().numpy(), 0, note)
        Qf = D.form_q(dA, handle=hc)[:, :UNITS].cpu().numpy()
        for j in range(UNITS):
            check_solve(label, ref, "qb", Qf[:, j], E.RHS + j, f"form_q column {j}; {note}")
        # the minimum-norm solution of A'y = c against tests/adjoint_ext.c, judged like x
        c = F.rhs(n, 1, seed=3)
        _, y_e = AO.adj_ext(ref.A, c)
        y64 = AO.np_solve_adj(ref.H64, ref.a64, c)
        del ref.H64
        yd = torch.zeros(m, dtype=torch.float64, device=DEV)
        yd[:n] = torch.from_numpy(c).to(DEV)
        y = D.solve_adjoint_(yd.clone(), dA, st.α, handle=hc).cpu().numpy()
        s = E.nrm(y_e)
        TABLE.check(f"solve_adjoint_ m={mname}", ref, {"x": E.nrm(y - y_e) / s}, {"x": E.nrm(y64 - y_e) / s}, note=note)
        record_memory(m, family, free0)
        check_switch(m, {
            "apply_qt_": qt_dot_launches(hc, lambda: D.apply_qt_(b0.clone(), dA, handle=hc)),
            "apply_q_": qt_dot_launches(hc, lambda: D.apply_q_(b0.clone(), dA, handle=hc)),
            "ldiv": qt_dot_launches(hc, lambda: D.ldiv(H, b0)),
            "solve_adjoint_": qt_dot_launches(hc, lambda: D.solve_adjoint_(yd.clone(), dA, st.α, handle=hc)),
        })
    finally:
        torch.cuda.synchronize()
        hc.close()


@pytest.mark.parametrize("family", MILLION_FAMILIES)
@pytest.mark.parametrize("mname", list(MILLION))
def test_million_rows_qrcp(D, coracle, mname, family):
    m, n = MILLION[mname], MILLION_N
    hc, free0 = fresh_handle(D, m)
    try:
        A0 = F.make(family, m, n)
        dA = D.to_colmajor(A0, DEV)
        st = D.qrcp_(dA, handle=hc)
        torch.cuda.synchronize()
        H, alpha, p = npy(st.A), st.α.cpu().numpy(), st.p.cpu().numpy()
        assert sorted(p) == list(range(n))
        # the rule on A[:, p] (test_gpu_qrcp.py::check_factor); its right-hand sides give the basic solution at full rank
        ref = E.Ref(coracle, None, family, m, n, A=np.asfortranarray(A0[:, p]), keep_h64=True)
        label, note = f"qrcp m={mname}", f"qrcp {m}x{n}"
        gpu, absolute = E.factor_checks(label, ref, H, alpha, note)
        TABLE.check(label, ref, gpu, ref.e64, absolute, note)
        del H
        b0 = torch.from_numpy(ref.b[:, 0].copy()).to(DEV)
        x = D.solve_qrcp_(b0.clone(), st.A, st.α, st.p, n, handle=hc).cpu().numpy()
        check_solve(f"solve_qrcp_ m={mname}", ref, "x", x[p], 0, f"nrhs=1; {note}")
        Bd = D.to_colmajor(ref.b[:, 1:4], DEV)
        X = D.solve_qrcp_(Bd, st.A, st.α, st.p, n, handle=hc).cpu().numpy()
        for r in range(1, 4):
            check_solve(f"solve_qrcp_ m={mname}", ref, "x", X[p, r - 1], r, f"nrhs=3; {note}")
        # the minimum-norm solution against the long-double twin (tests/cod_ext.c) with the device's permutation
        bh = ref.b[:, 0].copy()
        fac = (ref.H64, ref.a64, p)
        floor = E.FLOOR_EPS * E.EPS * E.SIZE["x"](m)
        cod = {}
        for r in (n, n // 2):
            Fd, gd = D.cod_(st.A, st.α, r, handle=hc)
            cod[r] = (Fd, gd)
            xd = D.solve_cod_(b0.clone(), st.A, st.p, Fd, gd, r, handle=hc).cpu().numpy()
            x_ext = CM.cod_ext(A0, p, r, bh)
            x64 = CM.cod_fp64(coracle, A0, bh, r, fac)[0]
            s = E.nrm(x_ext)
            got, e64 = E.nrm(xd - x_ext) / s, E.nrm(x64 - x_ext) / s
            TABLE.check(f"solve_cod_ m={mname} rank={'n' if r == n else 'n/2'}", ref, {"x": got}, {"x": e64}, note=note)
            assert got <= E.C_REL * max(e64, floor)
        record_memory(m, family, free0)
        check_switch(m, {
            "solve_qrcp_": qt_dot_launches(hc, lambda: D.solve_qrcp_(b0.clone(), st.A, st.α, st.p, n, handle=hc)),
            "solve_cod_": qt_dot_launches(hc, lambda: D.solve_cod_(b0.clone(), st.A, st.p, *cod[n], n, handle=hc)),
        })
    finally:
        torch.cuda.synchronize()
        hc.close()
