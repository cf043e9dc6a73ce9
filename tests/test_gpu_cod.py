"""The complete orthogonal decomposition on the pivoted QR (dhqr_cod_f64) and the minimum-norm solution at a given rank
(dhqr_solve_cod_f64), DESIGN §2.8.

dhqr_cod_f64 is the unpivoted factorisation of R_r' (n x r) built from the device's own pivoted R, so its accuracy yardstick is
the extended-precision rule of ext_rule.py on that matrix.  The solve is held to the same rule against the long-double twin of
the whole computation (tests/cod_model.py: cod_ext) with the device's permutation and rank, with the fp64 twin on the same
permutation as the comparison.  On top of it: the minimum-norm property (SVD pseudo-inverse, null space, the basic solution),
the shape edges, a refused wide panel of R_r', composability with form_q / forwardsolve_ / apply_q_, right-hand-side widths,
and the storage, stream, launch-accounting, memory and argument contracts.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import cod_model as CM
import ext_rule as E
import matrix_families as F
from test_gpu_qrcp import _outside, _placed
from test_gpu_streams import STREAM_KINDS, Case, Gate, P, SP, dev, run_gated

DEV = "cuda:0"
FAMILIES = tuple(f for f in F.FAMILIES if f not in F.NAN_FAMILIES)
TABLE = E.Table("cod_ext.md")


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
    TABLE.write()


def npy(t):
    return np.asfortranarray(t.cpu().numpy())


def qrcp(D, h, A0):
    A = D.to_colmajor(A0, DEV)
    st = D.qrcp_(A, handle=h)
    torch.cuda.synchronize()
    return st, npy(st.A), st.α.cpu().numpy(), st.p.cpu().numpy()


def solve(D, h, st, r, b, **opts):
    """(x, F, gamma) on the device at rank r for the (m, k) block b."""
    with E.options(h, **opts):
        Fd, gd = D.cod_(st.A, st.α, r, handle=h)
        db = D.to_colmajor(b, DEV)
        D.solve_cod_(db, st.A, st.p, Fd, gd, r, handle=h)
        torch.cuda.synchronize()
    return db.cpu().numpy(), Fd, gd


def check_x(coracle, A0, H, alpha, p, r, b, x, where):
    """err_gpu <= C_REL max(err_fp64_twin, floor) against the long-double twin, per right-hand side; the fp64 twin factors
    A[:, p] unpivoted in fp64, so both twins use the device's permutation and rank."""
    m, n = A0.shape
    x_ext = CM.cod_ext(A0, p, r, b)
    H64, a64 = coracle.qr(np.asfortranarray(A0[:, p]))
    x64 = CM.cod_fp64(coracle, A0, b, r, (H64, a64, p))[0]
    floor = E.FLOOR_EPS * E.EPS * E.SIZE["x"](m)
    for k in range(b.shape[1]):
        scale = E.nrm(x_ext[:, k])
        got, e64 = E.nrm(x[:n, k] - x_ext[:, k]) / scale, E.nrm(x64[:, k] - x_ext[:, k]) / scale
        assert got <= E.C_REL * max(e64, floor), f"x: {got:.3e} vs fp64 twin {e64:.3e}; rhs {k}; {where}"


def rhs(m, k, seed=5):
    return np.asfortranarray(F.rhs(m, k, seed=seed).reshape(m, k))


# ---------------------------------------------------------------------------------------------------------------------
# 1: the second factorisation on the device's own R_r'
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_cod_factor_families(D, h, coracle, family):
    A0 = F.make(family, 2048, 512)
    st, H, alpha, p = qrcp(D, h, A0)
    r = st.rank()
    assert r > 0
    Fd, gd = D.cod_(st.A, st.α, r, handle=h)
    torch.cuda.synchronize()
    assert tuple(Fd.shape) == (512, r) and tuple(gd.shape) == (r,)
    ref = E.Ref(coracle, None, family, 512, r, A=CM.rr_t(H, alpha, r), solve=False)
    gpu, absolute = E.factor_checks("cod", ref, npy(Fd), gd.cpu().numpy(), f"R_r' of qrcp {A0.shape}, rank {r}")
    TABLE.check("cod", ref, gpu, ref.e64, absolute)


# ---------------------------------------------------------------------------------------------------------------------
# 2-3: the minimum-norm solution end to end
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 31, 32, 33, 37, 128, 129, 255, 256])
@pytest.mark.parametrize("noisy", [False, True])
def test_solve_cod_low_rank(D, h, coracle, r, noisy):
    m, n = 2048, 256
    A0 = CM.low_rank(m, n, r, 1e-13 if noisy else 0.0)
    st, H, alpha, p = qrcp(D, h, A0)
    rd = st.rank(rcond=1e-8)
    assert rd == r
    b = rhs(m, 1)
    x, _, _ = solve(D, h, st, rd, b)
    check_x(coracle, A0, H, alpha, p, rd, b, x, f"rank {r}{' noisy' if noisy else ''}")


@pytest.mark.gpu
@pytest.mark.parametrize("r", [37, 128, 200])
def test_solve_cod_minimum_norm(D, h, r):
    m, n = 2048, 256
    A0 = CM.low_rank(m, n, r)
    b = F.rhs(m, 1, seed=7)
    st = D.qrcp_(D.to_colmajor(A0, DEV), handle=h)
    assert st.rank() == r
    cs = st.cod()
    assert cs.rank == r and cs.qrcp is st and cs.F is not None and cs.gamma is cs.γ
    A_before, p_before = st.A.clone(), st.p.clone()
    bd = torch.from_numpy(b).to(DEV)
    x = cs.ldiv(bd).cpu().numpy()
    assert torch.equal(st.A, A_before) and torch.equal(st.p, p_before) and torch.equal(bd.cpu(), torch.from_numpy(b))
    x_pinv = CM.pinv_solve(A0, b, r)
    assert np.linalg.norm(x - x_pinv) <= 1e-8 * np.linalg.norm(x_pinv)
    Nul = np.linalg.svd(A0)[2][r:].T                                 # null-space basis of the exactly rank-r A
    assert np.linalg.norm(Nul.T @ x) <= 1e-10 * np.linalg.norm(x)
    xb, rb = st.ldiv(bd)                                              # the basic solution: unchanged behaviour
    xb = xb.cpu().numpy()
    assert rb == r
    res, resb = np.linalg.norm(A0 @ x - b), np.linalg.norm(A0 @ xb - b)
    assert abs(res - resb) <= 1e-10 * np.linalg.norm(b)
    assert np.linalg.norm(x) <= np.linalg.norm(xb)


# ---------------------------------------------------------------------------------------------------------------------
# 4: edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_solve_cod_full_rank_matches_basic(D, h, coracle):
    m, n = 1500, 200
    A0 = F.make("normal", m, n)
    st, H, alpha, p = qrcp(D, h, A0)
    b = rhs(m, 2)
    x, _, _ = solve(D, h, st, n, b)
    check_x(coracle, A0, H, alpha, p, n, b, x, "rank n")
    db = D.to_colmajor(b, DEV)
    xq = D.solve_qrcp_(db, st.A, st.α, st.p, n, handle=h).cpu().numpy()
    assert np.abs(x[:n] - xq).max() <= 1e-12 * np.abs(xq).max()


@pytest.mark.gpu
def test_solve_cod_rank_zero(D, h):
    m, n, nrhs = 400, 100, 2
    st = D.qrcp_(D.to_colmajor(F.make("normal", m, n), DEV), handle=h)
    Fbuf = torch.full((n * 3,), float("nan"), dtype=torch.float64, device=DEV)
    gbuf = torch.full((8,), float("nan"), dtype=torch.float64, device=DEV)
    cur = SP(torch.cuda.current_stream())
    D._lib.call("dhqr_cod_f64", h.raw, m, n, 0, P(st.A), m, P(st.α), P(Fbuf), n, P(gbuf), cur)
    b = D.to_colmajor(rhs(m, nrhs), DEV)
    b0 = b.clone()
    D._lib.call("dhqr_solve_cod_f64", h.raw, m, n, 0, P(st.A), m, P(st.p), P(Fbuf), n, P(gbuf), P(b), m, nrhs, cur)
    torch.cuda.synchronize()
    assert torch.isnan(Fbuf).all() and torch.isnan(gbuf).all()
    assert not b[:n].any() and torch.equal(b[n:], b0[n:])
    Fd, gd = D.cod_(st.A, st.α, 0, handle=h)
    assert tuple(Fd.shape) == (n, 0) and tuple(gd.shape) == (0,)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,r", [(1, 1, 1), (33, 32, 1), (33, 32, 32), (300, 128, 127), (300, 128, 128), (300, 129, 128),
                                   (300, 160, 128), (300, 161, 128), (300, 160, 129), (400, 257, 129), (400, 129, 1), (300, 64, 33)])
def test_solve_cod_shape_edges(D, h, coracle, m, n, r):
    A0 = CM.low_rank(m, n, r) if r < n else F.make("normal", m, n)
    st, H, alpha, p = qrcp(D, h, A0)
    b = rhs(m, 1)
    x, Fd, gd = solve(D, h, st, r, b)
    check_x(coracle, A0, H, alpha, p, r, b, x, f"{m}x{n} rank {r}")
    ref = E.Ref(coracle, None, "lowrank", n, r, A=CM.rr_t(H, alpha, r), solve=False)
    gpu, absolute = E.factor_checks("cod edges", ref, npy(Fd), gd.cpu().numpy(), f"R_r' of {m}x{n}, rank {r}")
    TABLE.check("cod edges", ref, gpu, ref.e64, absolute)


@pytest.mark.gpu
def test_cod_refused_wide_panel(D, h, coracle):
    """R_r' has a full 128-column panel; with the chain's conditioning guard (option "wide_kappa") tightened below what any
    128-column panel meets, the wide chain turns it down, the factorisation is redone by the 32-column chain from that panel on,
    and the result is still held to the rule."""
    m, n, r = 1200, 400, 300
    A0 = CM.low_rank(m, n, r, 1e-13)
    st, H, alpha, p = qrcp(D, h, A0)
    c0 = E.counters(h)
    h.set_option("wide_kappa", 1)
    try:
        b = rhs(m, 1)
        x, Fd, gd = solve(D, h, st, r, b)
    finally:
        h.set_option("wide_kappa", 1000)
    c1 = E.counters(h)
    assert c1["wide_redone"] > c0["wide_redone"], (c0, c1)
    check_x(coracle, A0, H, alpha, p, r, b, x, "refused wide panel")
    ref = E.Ref(coracle, None, "lowrank", n, r, A=CM.rr_t(H, alpha, r), solve=False)
    gpu, absolute = E.factor_checks("cod refused", ref, npy(Fd), gd.cpu().numpy(), f"counters {c0} -> {c1}")
    TABLE.check("cod refused", ref, gpu, ref.e64, absolute)


# ---------------------------------------------------------------------------------------------------------------------
# 5: composability and right-hand sides
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cod_composes(D, h):
    m, n, r = 1200, 300, 260
    A0 = CM.low_rank(m, n, r)
    st, H, alpha, p = qrcp(D, h, A0)
    Fd, gd = D.cod_(st.A, st.α, r, handle=h)
    Z = D.form_q(Fd, handle=h)
    U = D.form_r(Fd, gd)
    RrT = torch.from_numpy(CM.rr_t(H, alpha, r)).to(DEV)
    assert float((Z.T @ Z - torch.eye(r, dtype=torch.float64, device=DEV)).abs().max()) < 1e-13
    assert float((Z @ U - RrT).norm() / RrT.norm()) < 1e-13
    # the inner stage of dhqr_solve_cod_f64 is forwardsolve_ and apply_q_ on (F, gamma): bitwise the same x
    b = torch.from_numpy(F.rhs(m, 1, seed=3)).to(DEV)
    c = D.apply_qt_(b.clone(), st.A[:, :r], handle=h)                 # the first r reflectors
    y = torch.zeros(n, dtype=torch.float64, device=DEV)
    y[:r] = c[:r]
    D.forwardsolve_(y, Fd, gd, handle=h)
    D.apply_q_(y, Fd, handle=h)
    xs = torch.zeros(n, dtype=torch.float64, device=DEV)
    xs[st.p] = y
    s = b.clone()
    D.solve_cod_(s, st.A, st.p, Fd, gd, r, handle=h)
    torch.cuda.synchronize()
    assert torch.equal(s[:n], xs)
    assert torch.equal(s[n:], c[n:])                                  # rows n..m-1: H_r ... H_1 b


@pytest.mark.gpu
@pytest.mark.parametrize("nrhs", [1, 3, 65])
@pytest.mark.parametrize("qt_vec", [1, 0])
def test_solve_cod_rhs_widths(D, h, coracle, nrhs, qt_vec):
    m, n, r = 1500, 200, 150
    A0 = CM.low_rank(m, n, r)
    st, H, alpha, p = qrcp(D, h, A0)
    b = rhs(m, nrhs)
    with E.options(h, qt_vec=qt_vec):
        Fd, gd = D.cod_(st.A, st.α, r, handle=h)
        db = D.colmajor_empty(m, nrhs, DEV, lda=m + 3)
        db.copy_(torch.from_numpy(b))
        D.solve_cod_(db, st.A, st.p, Fd, gd, r, handle=h)
        torch.cuda.synchronize()
    check_x(coracle, A0, H, alpha, p, r, b, db.cpu().numpy(), f"nrhs {nrhs}, qt_vec {qt_vec}, ldb m+3")


# ---------------------------------------------------------------------------------------------------------------------
# 6: contracts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cod_storage_contract(D, h):
    m, n, nrhs, r = 1100, 150, 3, 140
    st = D.qrcp_(D.to_colmajor(F.make("graded6", m, n), DEV), handle=h)
    torch.cuda.synchronize()
    A0, al0, p0 = st.A.clone(), st.α.clone(), st.p.clone()
    b0 = torch.from_numpy(np.asfortranarray(F.rhs(m, nrhs, seed=9))).to(DEV)
    cur = SP(torch.cuda.current_stream())
    results = []
    for lda, ldf, ldb in ((m, n, m), (m + 1, n + 1, m + 1), (m + 2, n + 3, m + 5)):
        for off in (0, 1):                                             # base 8 B off a 16 B boundary
            abuf, Av = _placed(A0, lda, off)
            albuf, alv = _placed(al0.reshape(n, 1), n, off)
            pbuf = torch.full((64 + off + n + 64,), -7, dtype=torch.int64, device=DEV)
            pv = pbuf[64 + off:64 + off + n]
            pv.copy_(p0)
            fbuf, Fv = _placed(torch.zeros(n, r, dtype=torch.float64, device=DEV), ldf, off)
            gbuf, gv = _placed(torch.zeros(r, 1, dtype=torch.float64, device=DEV), r, off)
            bbuf, bv = _placed(b0, ldb, off)
            inputs = (abuf.clone(), albuf.clone(), pbuf.clone())
            f_before, g_before, b_before = fbuf.clone(), gbuf.clone(), bbuf.clone()
            D._lib.call("dhqr_cod_f64", h.raw, m, n, r, P(Av), lda, P(alv), P(Fv), ldf, P(gv), cur)
            D._lib.call("dhqr_solve_cod_f64", h.raw, m, n, r, P(Av), lda, P(pv), P(Fv), ldf, P(gv), P(bv), ldb, nrhs, cur)
            torch.cuda.synchronize()
            where = f"lda {lda}, ldf {ldf}, ldb {ldb}, offset {off}"
            for buf, before in zip((abuf, albuf, pbuf), inputs):
                assert torch.equal(buf.view(torch.uint8), before.view(torch.uint8)), f"an input changed; {where}"
            for buf, before, ld, rows, k in ((fbuf, f_before, ldf, n, r), (gbuf, g_before, r, r, 1), (bbuf, b_before, ldb, m, nrhs)):
                mask = _outside(buf, off, ld, rows, k)
                assert torch.equal(buf[mask].view(torch.uint8), before[mask].view(torch.uint8)), f"wrote outside; {where}"
            results.append((where, Fv.clone(), gv.clone(), bv.clone()))
    for where, *rs in results[1:]:
        for a, b in zip(rs, results[0][1:]):
            assert np.ascontiguousarray(a.cpu().numpy()).tobytes() == np.ascontiguousarray(b.cpu().numpy()).tobytes(), \
                f"not bitwise equal; {where}"


@pytest.mark.gpu
def test_cod_repeatable(D, h):
    A0 = CM.low_rank(3000, 400, 300, 1e-13)
    st = D.qrcp_(D.to_colmajor(A0, DEV), handle=h)
    b = rhs(3000, 2)
    outs = [solve(D, h, st, 300, b) for _ in range(2)]
    digests = [E.digest(x, npy(Fd), gd.cpu().numpy()) for x, Fd, gd in outs]
    assert digests[0] == digests[1]


@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    return Gate()


@pytest.fixture(scope="module")
def streams():
    return {"nonblocking": torch.cuda.Stream(), "high": torch.cuda.Stream(priority=-100), "low": torch.cuda.Stream(priority=100),
            "legacy": torch.cuda.default_stream()}


def cod_case(D, h, name):
    m, n, r, nrhs = 700, 300, 260, 2                                  # R_r' (300 x 260) has two full 128-column panels
    sts = [D.qrcp_(D.to_colmajor(CM.low_rank(m, n, r, 1e-13, seed=s), DEV), handle=h) for s in (0, 1)]
    torch.cuda.synchronize()
    bufs = {"A": tuple(s.A.t().contiguous().reshape(-1) for s in sts), "alpha": tuple(s.α.clone() for s in sts),
            "p": tuple(s.p.clone() for s in sts)}
    if name == "cod":
        bufs["F"] = (torch.zeros(n * r, dtype=torch.float64, device=DEV), torch.full((n * r,), -1.0, dtype=torch.float64, device=DEV))
        bufs["gamma"] = (torch.zeros(r, dtype=torch.float64, device=DEV), torch.full((r,), -1.0, dtype=torch.float64, device=DEV))

        def fn(w, st):
            D._lib.call("dhqr_cod_f64", h.raw, m, n, r, P(w["A"]), m, P(w["alpha"]), P(w["F"]), n, P(w["gamma"]), st)
        return Case(fn, bufs, ("F", "gamma", "A", "alpha"))
    fac = [D.cod_(s.A, s.α, r, handle=h) for s in sts]
    torch.cuda.synchronize()
    bufs["F"] = tuple(f.t().contiguous().reshape(-1) for f, _ in fac)
    bufs["gamma"] = tuple(g.clone() for _, g in fac)
    bufs["b"] = (dev(np.asfortranarray(F.rhs(m, nrhs, seed=0))), dev(np.asfortranarray(F.rhs(m, nrhs, seed=1))))

    def fn(w, st):
        D._lib.call("dhqr_solve_cod_f64", h.raw, m, n, r, P(w["A"]), m, P(w["p"]), P(w["F"]), n, P(w["gamma"]), P(w["b"]), m, nrhs, st)
    return Case(fn, bufs, ("b", "A", "p", "F", "gamma"))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAM_KINDS)
@pytest.mark.parametrize("name", ["cod", "solve_cod"])
def test_cod_gated(D, h, gate, streams, name, kind):
    case = cod_case(D, h, name)
    case.reference(h)
    if name == "cod":
        assert case.delta["wide_panels"] > 0, "R_r' went around the wide chain: the synchronising path is not exercised"
    run_gated(case, gate, streams[kind], f"{name} on a {kind} stream")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cod_f64", "solve_cod_f64"])
def test_cod_profile_counts_every_launch(D, name):
    hd = D.Handle(0)
    try:
        hd.set_option("profile", 1)
        m, n, r, nrhs = 1024, 300, 260, 2
        st = D.qrcp_(D.to_colmajor(CM.low_rank(m, n, r, 1e-13), DEV), handle=hd)
        Fd, gd = D.cod_(st.A, st.α, r, handle=hd)
        b = D.to_colmajor(rhs(m, nrhs), DEV)
        torch.cuda.synchronize()
        hd.profile_reset()
        n0 = hd.launch_count()
        if name == "cod_f64":
            D.cod_(st.A, st.α, r, handle=hd)
        else:
            D.solve_cod_(b, st.A, st.p, Fd, gd, r, handle=hd)
        torch.cuda.synchronize()
        launched = hd.launch_count() - n0
        prof = hd.profile()
        assert launched > 0
        assert all(prof), f"a profile class without a name: {sorted(prof)}"
        counts = {k: v["count"] for k, v in prof.items() if v["count"]}
        assert sum(counts.values()) == launched, f"{launched} launches, profile counts {counts}"
        if name == "cod_f64":
            assert counts.get("k_cod_pack") == 1, counts
    finally:
        hd.close()


@pytest.mark.gpu
def test_cod_handle_returns_its_device_memory(D):
    m, n, r, nrhs = 16384, 1024, 1000, 3
    A0 = D.colmajor_empty(m, n, DEV)
    D.fill_uniform_(A0, 11)
    A, b, b0 = D.colmajor_empty(m, n, DEV), D.colmajor_empty(m, nrhs, DEV), D.colmajor_empty(m, nrhs, DEV)
    D.fill_uniform_(b0, 12)
    al = torch.zeros(n, dtype=torch.float64, device=DEV)
    jp = torch.zeros(n, dtype=torch.int64, device=DEV)
    Fm = D.colmajor_empty(n, r, DEV)
    g = torch.zeros(r, dtype=torch.float64, device=DEV)

    def run(hd):
        call = D._lib.call
        A.copy_(A0)
        call("dhqr_qrcp_f64", hd.raw, m, n, P(A), m, P(al), P(jp), None)
        call("dhqr_cod_f64", hd.raw, m, n, r, P(A), m, P(al), P(Fm), n, P(g), None)
        for k in (1, nrhs):
            b.copy_(b0)
            call("dhqr_solve_cod_f64", hd.raw, m, n, r, P(A), m, P(jp), P(Fm), n, P(g), P(b), m, k, None)
        torch.cuda.synchronize()

    def free_bytes():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info()[0]

    hd = D.Handle(0)
    try:
        run(hd)
    finally:
        hd.close()
    base = free_bytes()
    drift = []
    for _ in range(2):
        hd = D.Handle(0)
        try:
            run(hd)
        finally:
            hd.close()
        drift.append(base - free_bytes())
    assert all(d <= 16 << 20 for d in drift), "free memory below its baseline: " + ", ".join(f"{d / 2**20:.1f} MiB" for d in drift)


class _NullHandle:
    raw = C.c_void_p()


@pytest.mark.gpu
def test_cod_errors(D, h):
    m, n, r = 40, 30, 20
    A = D.to_colmajor(F.make("normal", m, n), DEV)
    alpha = torch.zeros(n + 1, dtype=torch.float64, device=DEV)
    p = torch.zeros(n + 1, dtype=torch.int64, device=DEV)
    Fm = torch.zeros(n * r + 1, dtype=torch.float64, device=DEV)
    g = torch.zeros(r + 1, dtype=torch.float64, device=DEV)
    b = D.to_colmajor(np.zeros((m + 1, 2)), DEV)
    st = SP(torch.cuda.current_stream())
    odd = lambda t: C.c_void_p(t.data_ptr() + 4)
    at = lambda t, k: C.c_void_p(t.data_ptr() + 8 * k)

    def code(fn, *args):
        with pytest.raises(D._lib.DhqrError) as e:
            D._lib.call(fn, *args)
        return e.value.code

    torch.cuda.synchronize()
    before = h.launch_count()
    snap = [t.clone() for t in (A, alpha, p, Fm, g, b)]
    cod = [h.raw, m, n, r, P(A), m, P(alpha), P(Fm), n, P(g), st]

    def bad(args, fn, i, v):
        a = list(args)
        a[i] = v
        return code(fn, *a)
    c = lambda i, v: bad(cod, "dhqr_cod_f64", i, v)
    assert c(0, None) == -1
    assert c(1, -1) == -2
    assert c(2, -1) == -3 and c(2, m + 1) == -3
    big = 728 * h.get_option("sms") + 1000                             # R_r' taller than the unpivoted path's row limit
    assert code("dhqr_cod_f64", h.raw, big, big, 1, P(A), big, P(alpha), P(Fm), big, P(g), st) == -3
    assert c(3, -1) == -4 and c(3, n + 1) == -4
    assert c(4, None) == -5 and c(4, odd(A)) == -5
    assert c(5, m - 1) == -6
    assert c(6, None) == -7 and c(6, odd(alpha)) == -7
    assert c(7, None) == -8 and c(7, odd(Fm)) == -8
    assert c(7, at(A, 5)) == -8 and c(7, at(alpha, 3)) == -8          # F over A's m x n block, over alpha
    assert c(8, n - 1) == -9
    assert c(9, None) == -10 and c(9, odd(g)) == -10
    assert c(9, at(A, m * n - 1)) == -10 and c(9, at(alpha, n - 1)) == -10 and c(9, at(Fm, n * r - 1)) == -10
    sv = [h.raw, m, n, r, P(A), m, P(p), P(Fm), n, P(g), P(b), m + 1, 2, st]
    s = lambda i, v: bad(sv, "dhqr_solve_cod_f64", i, v)
    assert s(0, None) == -1
    assert s(1, -1) == -2
    assert s(2, -1) == -3 and s(2, m + 1) == -3
    assert s(3, -1) == -4 and s(3, n + 1) == -4
    assert s(4, None) == -5 and s(4, odd(A)) == -5
    assert s(5, m - 1) == -6
    assert s(6, None) == -7 and s(6, odd(p)) == -7
    assert s(7, None) == -8 and s(7, odd(Fm)) == -8
    assert s(8, n - 1) == -9
    assert s(9, None) == -10 and s(9, odd(g)) == -10
    assert s(10, None) == -11 and s(10, odd(b)) == -11
    assert s(11, m - 1) == -12
    assert s(12, -1) == -13
    torch.cuda.synchronize()
    assert h.launch_count() == before, "a rejected call enqueued work"
    for t, t0 in zip((A, alpha, p, Fm, g, b), snap):
        assert torch.equal(t, t0)
    D._lib.call("dhqr_cod_f64", h.raw, 0, 0, 0, None, 1, None, None, 1, None, st)                    # n = 0
    D._lib.call("dhqr_cod_f64", h.raw, m, n, 0, P(A), m, P(alpha), None, n, None, st)               # rank = 0
    D._lib.call("dhqr_solve_cod_f64", h.raw, m, n, r, P(A), m, P(p), P(Fm), n, P(g), None, m, 0, st)  # nrhs = 0
    torch.cuda.synchronize()
    assert h.launch_count() == before, "a no-op enqueued work"
    with pytest.raises(D._lib.DhqrError) as e:
        D.cod_(A, alpha[:n], r, handle=_NullHandle())
    assert e.value.code == -1
