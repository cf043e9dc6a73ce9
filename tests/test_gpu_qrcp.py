"""QR with column pivoting on the device (dhqr_qrcp_f64) and the basic solution at a given rank (dhqr_solve_qrcp_f64).

A P = Q R is the unpivoted factorisation of A[:, p], so the accuracy yardstick is the extended-precision rule of ext_rule.py on
A[:, p] with the device's permutation p.  On top of it: the pivot invariant, LAPACK dgeqp3's permutation on separated inputs,
rank revelation, exact deficiency, the basic solution, composability with the other entry points, a matrix taller than the
unpivoted path takes, the renorm counter, and the storage, stream and argument contracts.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import ext_rule as E
import matrix_families as F
import qrcp_model as M
from test_gpu_streams import STREAM_KINDS, Case, Gate, P, SP, dev, run_gated

DEV = "cuda:0"
FAMILIES = tuple(f for f in F.FAMILIES if f not in F.NAN_FAMILIES)
SEPARATED = ("colscale", "graded6", "graded12", "rowscale")
TABLE = E.Table("qrcp_ext.md")


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


def qrcp(D, h, A0, lda=None):
    A = D.colmajor_empty(*A0.shape, DEV, lda=lda)
    A.copy_(torch.from_numpy(A0))
    st = D.qrcp_(A, handle=h)
    torch.cuda.synchronize()
    return st, np.asfortranarray(A.cpu().numpy()), st.α.cpu().numpy(), st.p.cpu().numpy()


class PRef(E.Ref):
    """ext_rule.Ref of a given matrix (A[:, p]): extended and fp64 factorisations of its leading k columns, optionally with
    right-hand sides b (the extended least-squares solution of the leading k columns)."""

    def __init__(self, coracle, A, family, k=None, b=None):
        self.family, (self.m, self.n) = family, A.shape
        self.A = A
        self.nan_cols = self.nan_alpha = None
        self.k = k = self.n if k is None else k
        self.solve = b is not None
        Ak = np.asfortranarray(A[:, :k])
        self.cn = np.linalg.norm(Ak, axis=0)
        if b is not None:
            self.b = np.asfortranarray(b.reshape(self.m, -1))
            self.He, self.ae, _, _, self.x_e = coracle.qr_ext(Ak, self.b)
        else:
            self.He, self.ae = coracle.qr_ext(Ak)
        H64, a64 = coracle.qr(Ak.copy(order="F"))
        if b is not None:
            self.x64 = np.stack([coracle.ldiv(H64, a64, self.b[:, r].copy()) for r in range(self.b.shape[1])], 1)
        self.e64 = E.factor_errors(H64, a64, self)


def check_factor(coracle, path, family, A0, H, alpha, p, k=None):
    ref = PRef(coracle, np.asfortranarray(A0[:, p]), family, k)
    gpu, absolute = E.factor_checks(path, ref, H, alpha, f"qrcp {A0.shape}")
    TABLE.check(path, ref, gpu, ref.e64, absolute)


def tails(H, alpha):
    """tail[k, c] = ||R[k:c+1, c]||: the norm of column c after k reflectors, from the computed R."""
    R = M.form_r(H, alpha)
    return np.sqrt(np.cumsum((R * R)[::-1], axis=0)[::-1])


def check_pivot_invariant(H, alpha):
    t = tails(H, alpha)
    n = H.shape[1]
    for k in range(n - 1):
        if abs(alpha[k]) >= 1e-8 * abs(alpha[0]):
            assert alpha[k] ** 2 >= (1 - 1e-6) * t[k, k + 1:].max() ** 2, f"step {k}: a larger column was left behind"


# ---------------------------------------------------------------------------------------------------------------------
# 1-3: accuracy, the pivot invariant, LAPACK's pivots
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_qrcp_families(D, h, coracle, family):
    A0 = F.make(family, 2048, 512)
    _, H, alpha, p = qrcp(D, h, A0)
    assert sorted(p) == list(range(512))
    check_factor(coracle, "qrcp", family, A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n", [(200, 1), (300, 31), (300, 32), (300, 33), (500, 63), (500, 64), (500, 65), (65, 65), (66, 65),
                                 (33, 32), (1, 1)])
def test_qrcp_shape_edges(D, h, coracle, m, n):
    A0 = F.make("normal", m, n)
    _, H, alpha, p = qrcp(D, h, A0)
    check_factor(coracle, "qrcp", "normal", A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


@pytest.mark.gpu
@pytest.mark.parametrize("family", SEPARATED)
def test_qrcp_pivots_match_dgeqp3(D, h, family):
    A0 = F.make(family, 2048, 256)
    _, pl = M.dgeqp3_refformat(A0)[1:]
    _, H, alpha, p = qrcp(D, h, A0)
    assert np.array_equal(p, pl)


# ---------------------------------------------------------------------------------------------------------------------
# 4-5: rank revelation and exact deficiency
# ---------------------------------------------------------------------------------------------------------------------
def low_rank(m, n, r, noise=0.0, seed=3):
    rng = np.random.default_rng([m, n, r, seed])
    a = (F._orth(rng, m, r) * np.logspace(0, -3, r)) @ F._orth(rng, n, r).T
    if noise:
        a = a + noise * rng.standard_normal((m, n))
    return np.asfortranarray(a)


@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 37, 128, 255])
@pytest.mark.parametrize("noisy", [False, True])
def test_qrcp_rank_revealing(D, h, coracle, r, noisy):
    m, n = 2048, 256
    A0 = low_rank(m, n, r, 1e-13 if noisy else 0.0)
    st, H, alpha, p = qrcp(D, h, A0)
    if noisy:
        assert st.rank(rcond=1e-8) == r
        # the default rcond = max(m, n) eps sits far below noise of 1e-13: every column counts, which is right for this input
        assert st.rank() == n
    else:
        assert st.rank() == r
    check_factor(coracle, f"qrcp rank {r}{' noisy' if noisy else ''}", "lowrank", A0, H, alpha, p, k=r)


@pytest.mark.gpu
@pytest.mark.parametrize("family", F.NAN_FAMILIES)
def test_qrcp_zero_column(D, h, coracle, family):
    m, n = 2048, 512
    A0 = F.make(family, m, n)
    _, H, alpha, p = qrcp(D, h, A0)
    assert np.isfinite(H).all() and np.isfinite(alpha).all()
    assert p[-1] == F.zero_column(family, n) and alpha[-1] == 0.0 and not H[n - 1:, n - 1].any()
    assert E.backward_error(np.asfortranarray(A0[:, p[:n - 1]]), H, alpha) < 1e-13


@pytest.mark.gpu
def test_qrcp_zero_matrix_and_nan(D, h):
    _, H, alpha, p = qrcp(D, h, np.zeros((300, 70), order="F"))
    assert not H.any() and not alpha.any() and np.array_equal(p, np.arange(70))
    A0 = F.make("normal", 300, 70)
    A0[123, 45] = np.nan
    _, H, alpha, p = qrcp(D, h, A0)
    assert np.isnan(alpha[0])


# ---------------------------------------------------------------------------------------------------------------------
# 6: the basic solution
# ---------------------------------------------------------------------------------------------------------------------
def check_basic(D, h, coracle, A0, r, nrhs, where):
    m, n = A0.shape
    st, H, alpha, p = qrcp(D, h, A0)
    b = np.asfortranarray(F.rhs(m, nrhs, seed=5).reshape(m, nrhs))
    db = D.to_colmajor(b, DEV)
    D.solve_qrcp_(db, st.A, st.α, st.p, r, handle=h)
    x = db.cpu().numpy()[:n]
    assert not x[p[r:]].any(), f"x is not zero off the leading columns; {where}"
    if r == 0:
        return x
    ref = PRef(coracle, np.asfortranarray(A0[:, p[:r]]), "basic", b=b)
    for k in range(nrhs):
        got, e64 = ref.solve_errors("x", x[p[:r], k], k)
        floor = E.FLOOR_EPS * E.EPS * E.SIZE["x"](m)
        assert got <= E.C_REL * max(e64, floor), f"x: {got:.3e} vs fp64 {e64:.3e}; rhs {k}; {where}"
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 37, 128, 255])
def test_solve_qrcp_low_rank(D, h, coracle, r):
    check_basic(D, h, coracle, low_rank(2048, 256, r), r, 1, f"rank {r}")


@pytest.mark.gpu
@pytest.mark.parametrize("nrhs", [1, 3, 65])
def test_solve_qrcp_full_rank(D, h, coracle, nrhs):
    A0 = F.make("normal", 1500, 200)
    x = check_basic(D, h, coracle, A0, 200, nrhs, f"full rank, nrhs {nrhs}")
    # r = n: the same as dhqr_solve_f64 on A[:, p], permuted back
    st, H, alpha, p = qrcp(D, h, A0)
    b = D.to_colmajor(np.asfortranarray(F.rhs(1500, nrhs, seed=5).reshape(1500, nrhs)), DEV)
    y = D.solve_householder_(b, st.A, st.α, handle=h).cpu().numpy()
    assert np.abs(x[p] - y).max() <= 1e-12 * np.abs(y).max()


@pytest.mark.gpu
def test_solve_qrcp_rank_zero_and_bad_jpvt(D, h, coracle):
    m, n = 400, 100
    x = check_basic(D, h, coracle, F.make("normal", m, n), 0, 2, "rank 0")
    assert not x.any()
    st = D.qrcp_(D.to_colmajor(F.make("normal", m, n), DEV), handle=h)
    pbad = st.p.clone()
    pbad[3], pbad[10] = -1, n                                          # out of range: skipped
    buf = torch.full((m + 64,), float("nan"), dtype=torch.float64, device=DEV)
    b = buf[32:32 + m]
    b.copy_(torch.from_numpy(F.rhs(m, 1, seed=2)))
    D.solve_qrcp_(b, st.A, st.α, pbad, n, handle=h)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:32]).all() and torch.isnan(buf[32 + m:]).all()


# ---------------------------------------------------------------------------------------------------------------------
# 7: composability with the other entry points
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_qrcp_composes(D, h):
    m, n = 1200, 300
    A0 = F.make("graded6", m, n)
    st = D.qrcp_(D.to_colmajor(A0, DEV), handle=h)
    Ap = torch.from_numpy(np.ascontiguousarray(A0)).to(DEV)[:, st.p]
    R = D.form_r(st.A, st.α)
    Q = D.form_q(st.A, handle=h)
    assert float(((Q @ R - Ap).norm(dim=0) / Ap.norm(dim=0)).max()) < 1e-13
    b = torch.from_numpy(F.rhs(m, 1, seed=1)).to(DEV)
    w = D.apply_q_(D.apply_qt_(b.clone(), st.A, handle=h), st.A, handle=h)
    assert float((w - b).norm() / b.norm()) < 1e-13
    c = torch.zeros(m, dtype=torch.float64, device=DEV)
    c[:n] = torch.from_numpy(F.rhs(n, 1, seed=4)).to(DEV)
    z = D.forwardsolve_(c.clone(), st.A, st.α, handle=h)
    zr = torch.linalg.solve_triangular(R.T, c[:n].reshape(-1, 1), upper=False)[:, 0]
    assert float((z - zr).norm() / zr.norm()) < 1e-9


# ---------------------------------------------------------------------------------------------------------------------
# 8-9: taller than the unpivoted path's limit; renorms
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_qrcp_tall(D, h, coracle):
    m, n = 728 * h.get_option("sms") + 1000, 64
    A0 = F.make("normal", m, n)
    _, H, alpha, p = qrcp(D, h, A0)
    check_factor(coracle, "qrcp tall", "normal", A0, H, alpha, p)
    check_pivot_invariant(H, alpha)
    check_basic(D, h, coracle, A0, n, 1, "tall")


@pytest.mark.gpu
def test_qrcp_renorms(D, h, coracle):
    A0 = M.nearly_parallel(2048, 256)
    torch.cuda.synchronize()
    r0 = h.get_option("qrcp_renorms")
    _, H, alpha, p = qrcp(D, h, A0)
    assert h.get_option("qrcp_renorms") - r0 >= 1
    check_factor(coracle, "qrcp", "nearly_parallel", A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


# ---------------------------------------------------------------------------------------------------------------------
# 10: contracts
# ---------------------------------------------------------------------------------------------------------------------
def _placed(src, ld, off, pad=64, fill=float("nan")):
    m, k = src.shape
    buf = torch.full((pad + off + ld * k + pad,), fill, dtype=src.dtype, device=DEV)
    view = buf[pad + off:pad + off + ld * k].view(k, ld).t()[:m]
    view.copy_(src)
    return buf, view


def _outside(buf, off, ld, m, k, pad=64):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[pad + off:pad + off + ld * k].view(k, ld)[:, :m] = False
    return mask


@pytest.mark.gpu
def test_qrcp_storage_contract(D, h):
    m, n, nrhs, r = 1100, 150, 3, 140
    A0 = torch.from_numpy(F.make("graded6", m, n)).to(DEV)
    b0 = torch.from_numpy(np.asfortranarray(F.rhs(m, nrhs, seed=9))).to(DEV)
    results = []
    for lda in (m, m + 1, m + 2):
        for off in (0, 1):                                             # base 8 B off a 16 B boundary
            abuf, Av = _placed(A0, lda, off)
            albuf, alv = _placed(torch.zeros(n, 1, dtype=torch.float64, device=DEV), n, off)
            pbuf = torch.full((64 + off + n + 64,), -7, dtype=torch.int64, device=DEV)
            pv = pbuf[64 + off:64 + off + n]
            a_before, al_before, p_before = abuf.clone(), albuf.clone(), pbuf.clone()
            D._lib.call("dhqr_qrcp_f64", h.raw, m, n, P(Av), lda, P(alv), P(pv), SP(torch.cuda.current_stream()))
            bbuf, bv = _placed(b0, m + 1, off)
            b_before = bbuf.clone()
            D._lib.call("dhqr_solve_qrcp_f64", h.raw, m, n, r, P(Av), lda, P(alv), P(pv), P(bv), m + 1, nrhs,
                        SP(torch.cuda.current_stream()))
            torch.cuda.synchronize()
            where = f"lda {lda}, offset {off}"
            for buf, before, ld, k in ((abuf, a_before, lda, n), (albuf, al_before, n, 1), (bbuf, b_before, m + 1, nrhs)):
                mask = _outside(buf, off, ld, m if buf is not albuf else n, k)
                assert torch.equal(buf[mask].view(torch.uint8), before[mask].view(torch.uint8)), f"wrote outside; {where}"
            pm = torch.ones_like(pbuf, dtype=torch.bool)
            pm[64 + off:64 + off + n] = False
            assert torch.equal(pbuf[pm], p_before[pm]), f"wrote outside jpvt; {where}"
            results.append((where, Av.clone(), alv.clone(), pv.clone(), bv.clone()))
    for where, *rs in results[1:]:
        for a, b in zip(rs, results[0][1:]):
            assert np.ascontiguousarray(a.cpu().numpy()).tobytes() == np.ascontiguousarray(b.cpu().numpy()).tobytes(), \
                f"not bitwise equal; {where}"


@pytest.mark.gpu
def test_qrcp_repeatable(D, h):
    A0 = F.make("colscale", 3000, 400)
    outs = [qrcp(D, h, A0)[1:] for _ in range(2)]
    assert E.digest(*outs[0]) == E.digest(*outs[1])


@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    return Gate()


@pytest.fixture(scope="module")
def streams():
    return {"nonblocking": torch.cuda.Stream(), "high": torch.cuda.Stream(priority=-100), "low": torch.cuda.Stream(priority=100),
            "legacy": torch.cuda.default_stream()}


def qrcp_case(D, h, name):
    m, n, nrhs = 700, 96, 2
    if name == "qrcp":
        bufs = {"A": (dev(F.make("normal", m, n, 0)), dev(F.make("normal", m, n, 1))),
                "alpha": (torch.zeros(n, dtype=torch.float64, device=DEV), torch.full((n,), -1.0, dtype=torch.float64, device=DEV)),
                "p": (torch.zeros(n, dtype=torch.int64, device=DEV), torch.full((n,), 5, dtype=torch.int64, device=DEV))}

        def fn(w, st):
            D._lib.call("dhqr_qrcp_f64", h.raw, m, n, P(w["A"]), m, P(w["alpha"]), P(w["p"]), st)
        return Case(fn, bufs, ("A", "alpha", "p"))
    sts = [D.qrcp_(D.to_colmajor(F.make("normal", m, n, s), DEV), handle=h) for s in (0, 1)]
    torch.cuda.synchronize()
    bufs = {"A": tuple(s.A.t().contiguous().reshape(-1) for s in sts), "alpha": tuple(s.α.clone() for s in sts),
            "p": tuple(s.p.clone() for s in sts),
            "b": (dev(np.asfortranarray(F.rhs(m, nrhs, seed=0))), dev(np.asfortranarray(F.rhs(m, nrhs, seed=1))))}

    def fn(w, st):
        D._lib.call("dhqr_solve_qrcp_f64", h.raw, m, n, n - 3, P(w["A"]), m, P(w["alpha"]), P(w["p"]), P(w["b"]), m, nrhs, st)
    return Case(fn, bufs, ("b", "A", "alpha", "p"))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAM_KINDS)
@pytest.mark.parametrize("name", ["qrcp", "solve_qrcp"])
def test_qrcp_gated(D, h, gate, streams, name, kind):
    case = qrcp_case(D, h, name)
    case.reference(h)
    run_gated(case, gate, streams[kind], f"{name} on a {kind} stream")


class _NullHandle:
    raw = C.c_void_p()


@pytest.mark.gpu
def test_qrcp_errors(D, h):
    m, n = 40, 30
    A = D.to_colmajor(F.make("normal", m, n), DEV)
    alpha = torch.zeros(n + 1, dtype=torch.float64, device=DEV)
    p = torch.zeros(n + 1, dtype=torch.int64, device=DEV)
    b = D.to_colmajor(np.zeros((m + 1, 2)), DEV)
    st = SP(torch.cuda.current_stream())
    odd = lambda t: C.c_void_p(t.data_ptr() + 4)

    def code(fn, *args):
        with pytest.raises(D._lib.DhqrError) as e:
            D._lib.call(fn, *args)
        return e.value.code

    torch.cuda.synchronize()
    before = h.launch_count()
    snap = [t.clone() for t in (A, alpha, p, b)]
    q = "dhqr_qrcp_f64"
    assert code(q, None, m, n, P(A), m, P(alpha), P(p), st) == -1
    assert code(q, h.raw, -1, 0, P(A), m, P(alpha), P(p), st) == -2
    assert code(q, h.raw, m, -1, P(A), m, P(alpha), P(p), st) == -3
    assert code(q, h.raw, m, m + 1, P(A), m, P(alpha), P(p), st) == -3
    assert code(q, h.raw, m, n, None, m, P(alpha), P(p), st) == -4
    assert code(q, h.raw, m, n, odd(A), m, P(alpha), P(p), st) == -4
    assert code(q, h.raw, m, n, P(A), m - 1, P(alpha), P(p), st) == -5
    assert code(q, h.raw, m, n, P(A), m, None, P(p), st) == -6
    assert code(q, h.raw, m, n, P(A), m, odd(alpha), P(p), st) == -6
    assert code(q, h.raw, m, n, P(A), m, P(alpha), None, st) == -7
    assert code(q, h.raw, m, n, P(A), m, P(alpha), odd(p), st) == -7
    s = "dhqr_solve_qrcp_f64"
    args = [h.raw, m, n, n, P(A), m, P(alpha), P(p), P(b), m + 1, 2, st]

    def bad(i, v):
        a = list(args)
        a[i] = v
        return code(s, *a)
    assert bad(0, None) == -1
    assert bad(1, -1) == -2
    assert bad(2, m + 1) == -3
    assert bad(3, -1) == -4 and bad(3, n + 1) == -4
    assert bad(4, None) == -5 and bad(4, odd(A)) == -5
    assert bad(5, m - 1) == -6
    assert bad(6, None) == -7 and bad(6, odd(alpha)) == -7
    assert bad(7, None) == -8 and bad(7, odd(p)) == -8
    assert bad(8, None) == -9 and bad(8, odd(b)) == -9
    assert bad(9, m - 1) == -10
    assert bad(10, -1) == -11
    torch.cuda.synchronize()
    assert h.launch_count() == before, "a rejected call enqueued work"
    for t, t0 in zip((A, alpha, p, b), snap):
        assert torch.equal(t, t0)
    D._lib.call(q, h.raw, 0, 0, None, 1, None, None, st)                       # n = 0: nothing to do
    D._lib.call(s, h.raw, m, n, n, P(A), m, P(alpha), P(p), None, m, 0, st)     # nrhs = 0
    with pytest.raises(D._lib.DhqrError) as e:
        D.qrcp_(A, handle=_NullHandle())
    assert e.value.code == -1
