"""Rows into and out of many small triangles in one launch, their back-substitution and the rolling solver built on them
(dhqr_qr_append_batched_f64, dhqr_qr_downdate_batched_f64, dhqr_backsolve_batched_f64, BatchedStreamingLeastSquares; DESIGN §2.13).

Accuracy, per problem of a batch that holds one matrix of every non-NaN family of matrix_families: the append against the stacked
oracle by the extended-precision rule of ext_rule.py (R', V, and the fused Q~'[c; e] and x = R'^{-1} c' where the family solves),
the downdate against the long-double twin of downdate_model (the fp64 unblocked recurrence is the err_fp64 side).  Then the shape
grid on both sides of every cluster-size switch and at the size limit, the Gram identities, the fused right-hand sides against the
single-problem applies, the failure rule, the batched back-substitution, the rolling solver, and the contracts: bitwise
independence of the batch, the position, the layout and the handle's history, sentinels, a B above 2^31 bytes, side streams, graph
capture, launch counts and every error code.

The module registers the three entry points in test_gpu_history.py's catalogue at import (it sorts before that module)."""
import ctypes as C
import shutil
import types

import numpy as np
import pytest
import torch

import dist_loopback as L
import downdate_model as M
import ext_rule as E
import matrix_families as F
import test_gpu_history as HIST
from test_gpu_streams import P, SP, Gate, same_bits as _same_bits

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TABLE = E.Table("batched_update_ext.md")
DD_TABLE = E.Table("batched_downdate_ext.md")
FAMILIES = tuple(f for f in F.FAMILIES if f not in F.NAN_FAMILIES)
LIM, COLS, SLAB = 196608, 1024, 24576
NULL = C.c_void_p(None)


def D_():
    import dhqr_b200
    return dhqr_b200


def same_bits(a, b):
    return _same_bits(a.reshape(-1).contiguous(), b.reshape(-1).contiguous())


def finite_families(m, n):
    """The non-NaN families whose m x n matrix is finite (some are not defined at the smallest shapes)."""
    with np.errstate(all="ignore"):
        return [f for f in FAMILIES if np.isfinite(F.make(f, m, n)).all()]


def cluster_size(k, ncol):
    cs = 1
    while cs < 8 and -(-k // cs) * ncol > SLAB:
        cs *= 2
    return cs


# ---------------------------------------------------------------------------------------------------------------------
# the history catalogue: six problems of n = 24 on the diagonal blocks of the catalogue's factorisation X["H"]
# ---------------------------------------------------------------------------------------------------------------------
HB, HN, HK = 6, 24, 40


def _hist_tp(name, hyp):
    def run(h, s, X):
        R, al = HIST.up(X["H"]), HIST.up(X["alpha"][:HB * HN])
        B = HIST.up(np.asfortranarray(X["A"][:HK, :HB * HN]))       # problem 0 can remove them: rows of its block's columns
        vt, c, e = HIST.zeros(HB * HN), HIST.up(np.asfortranarray(np.tile(X["b3"][:HN], (1, HB)))), \
            HIST.up(np.asfortranarray(np.tile(X["b3"][:HK], (1, HB))))
        args = [h.raw, HN, HK, HB, HIST.P(R), HIST.M, HN * HIST.M + HN, HIST.P(al), HN, HIST.P(B), HK, HK * HN, HIST.P(vt), HN,
                HIST.P(c), HN, HN * 3, HIST.P(e), HK, HK * 3, 3]
        out = {"R": R, "alpha": al, "B": B, "vtop": vt, "c": c, "e": e}
        if hyp:
            info = HIST.zeros(HB, torch.int64)
            args.append(HIST.P(info))
            out["info"] = info
        HIST.call(name, *args, HIST.SP(s))
        return out
    return run


HIST.case("append_batched_r3", "dhqr_qr_append_batched_f64")(_hist_tp("dhqr_qr_append_batched_f64", False))
HIST.case("downdate_batched_r3", "dhqr_qr_downdate_batched_f64")(_hist_tp("dhqr_qr_downdate_batched_f64", True))


@HIST.case("backsolve_batched_r3", "dhqr_backsolve_batched_f64")
def _hist_backsolve(h, s, X):
    R, al = HIST.up(X["H"]), HIST.up(X["alpha"][:HB * HN])
    b = HIST.up(np.asfortranarray(np.tile(X["b3"][:HN], (1, HB))))
    HIST.call("dhqr_backsolve_batched_f64", h.raw, HN, HB, HIST.P(R), HIST.M, HN * HIST.M + HN, HIST.P(al), HN, HIST.P(b), HN, HN * 3, 3,
              HIST.SP(s))
    return {"b": b}


# ---------------------------------------------------------------------------------------------------------------------
# fixtures and helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def D():
    assert torch.cuda.is_available()
    return D_()


@pytest.fixture(scope="module")
def h(D):
    hd = D.Handle(0)
    yield hd
    torch.cuda.synchronize()
    hd.close()
    TABLE.write()
    DD_TABLE.write()


def npy(t):
    return np.asfortranarray(t.cpu().numpy())


def cm(D, arrs, ld=None):
    """(batch, rows, cols) column-major device batch of the given host matrices."""
    a0 = np.asarray(arrs[0])
    if a0.ndim == 1:
        arrs = [np.asarray(a)[:, None] for a in arrs]
        a0 = arrs[0]
    out = D.colmajor_empty_batched(len(arrs), a0.shape[0], a0.shape[1], DEV, lda=ld)
    for i, a in enumerate(arrs):
        out[i].copy_(torch.from_numpy(np.asarray(a, dtype=np.float64)))
    return out


def full(R, alpha):
    n = alpha.size
    return np.triu(R[:n, :n], 1) + np.diag(alpha)


def signed(R):
    d = np.sign(np.diag(R))
    d[d == 0] = 1.0
    return d[:, None] * R


def relerr(got, ref):
    s = np.abs(ref).max()
    return float(np.abs(got - ref).max() / s) if s > 0 else float(np.abs(got).max())


def tp_args(h, n, k, batch, R, ldr, sr, al, sal, B, ldb, sb, vt, svt, c=None, ldc=1, sc=0, e=None, lde=1, se=0, nrhs=0, info=None):
    """The arguments of dhqr_qr_append_batched_f64 (with ``info``: of the downdate) before the stream; tensors become pointers."""
    p = lambda t: NULL if t is None else (t if isinstance(t, C.c_void_p) else P(t))
    args = [h.raw, n, k, batch, p(R), ldr, sr, p(al), sal, p(B), ldb, sb, p(vt), svt, p(c), ldc, sc, p(e), lde, se, nrhs]
    if info is not None:
        args.append(p(info))
    return args


def ccopy(D, x):
    """A column-major copy of a (batch, rows, cols) batch."""
    return D.colmajor_empty_batched(*x.shape, DEV).copy_(x)


def poisoned(D, Q, n):
    """A copy of the batch Q whose n x n blocks keep only their strict upper triangle: NaN on and below the diagonal."""
    iu = torch.triu(torch.ones(Q.shape[1], Q.shape[2], dtype=torch.bool, device=DEV), 1)
    return ccopy(D, torch.where(iu, Q, torch.full_like(Q, float("nan"))))


# ---------------------------------------------------------------------------------------------------------------------
# 1. the append: the extended-precision rule per problem, fused right-hand sides and the back-substitution
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(33, 20), (129, 300), (3, 1)], ids=lambda s: f"n{s[0]}k{s[1]}")
def test_append_ext(D, h, coracle, oracle, shape):
    n, k = shape
    nrhs, m0 = 3, n + 5
    fams = finite_families(m0 + k, n)
    mats = [F.make(f, m0 + k, n) for f in fams]
    bs = [F.rhs(m0 + k, nrhs).reshape(m0 + k, nrhs) for _ in fams]
    Q = cm(D, [a[:m0] for a in mats])
    st = D.qr_batched_(Q, handle=h)
    c = cm(D, [b[:m0] for b in bs])
    D.apply_qt_batched_(c, Q, h)                       # c = (Q'b)[0:n] of the first n + 5 rows
    torch.cuda.synchronize()
    R0, a0, c0 = Q.cpu().numpy(), st.α.cpu().numpy(), c.cpu().numpy()
    cc = cm(D, [x[:n] for x in c0])
    B = cm(D, [a[m0:] for a in mats])
    e = cm(D, [b[m0:] for b in bs])
    t = D.append_rows_batched_(Q, st.α, B, cc, e, handle=h)
    # the back-substitution on R' with NaN in the diagonal and lower part of its storage
    Rn = poisoned(D, Q, n)
    x = ccopy(D, cc)
    D.backsolve_batched_(x, Rn, st.α, h)
    torch.cuda.synchronize()
    R1, a1, V2, vt, c1, e1, x1 = Q.cpu().numpy(), st.α.cpu().numpy(), t.B.cpu().numpy(), t.vtop.cpu().numpy(), cc.cpu().numpy(), \
        e.cpu().numpy(), x.cpu().numpy()
    for i, fam in enumerate(fams):
        Ri = full(R0[i], a0[i])
        S = np.asfortranarray(np.vstack([Ri, mats[i][m0:]]))
        rhs = np.asfortranarray(np.vstack([c0[i][:n], bs[i][m0:]]))
        ref = E.Ref(coracle, oracle, fam, n + k, n, A=S, b=rhs)
        H = np.zeros((n + k, n))
        H[:n] = np.triu(R1[i][:n], 1) + np.diag(vt[i])
        H[n:] = V2[i]
        gpu, absolute = E.factor_checks("append_batched", ref, H, a1[i], f"problem {i} n={n} k={k}")
        # err_fp64 is the larger of the oracle's and the single-problem append's (dhqr_qr_append_f64 on the same R and B): both run
        # the structured recurrence, whose rounding differs from the unblocked oracle's on the stacked matrix, and on a strongly
        # graded family a late column keeps only ~1e-10 of its norm, so either rounding is amplified a millionfold
        Ra, aa = D.to_colmajor(np.triu(R0[i][:n, :n], 1), DEV), torch.from_numpy(a0[i].copy()).to(DEV)
        ts = D.append_rows_((Ra, aa), D.to_colmajor(mats[i][m0:], DEV), handle=h)
        Hs = np.zeros((n + k, n))
        Hs[:n] = np.triu(npy(Ra), 1) + np.diag(ts.vtop.cpu().numpy())
        Hs[n:] = npy(ts.B)
        e_single = E.factor_errors(Hs, aa.cpu().numpy(), ref)
        e64 = {key: max(ref.e64[key], e_single[key]) for key in ref.e64}
        TABLE.check(f"append_batched n={n} k={k}", ref, gpu, e64, absolute)
        if not ref.solve:
            continue
        cs_, es_ = D.to_colmajor(c0[i][:n], DEV), D.to_colmajor(bs[i][m0:], DEV)
        ts.apply_qt_(cs_, es_)
        xs_ = cs_.clone()
        D.backsolve_(xs_, Ra, aa, handle=h)
        got, single = np.vstack([c1[i], e1[i]]), np.vstack([npy(cs_), npy(es_)])
        sc, sx = E.nrm(ref.b), E.nrm(ref.x_e)
        g = {"qtb": E.nrm(got - ref.qtb_e) / sc, "x": E.nrm(x1[i] - ref.x_e) / sx}
        e64 = {"qtb": max(E.nrm(ref.qtb64 - ref.qtb_e), E.nrm(single - ref.qtb_e)) / sc,
               "x": max(E.nrm(ref.x64 - ref.x_e), E.nrm(npy(xs_) - ref.x_e)) / sx}
        TABLE.check(f"append_batched n={n} k={k} nrhs 3", ref, g, e64, note=f"problem {i}: fused [c; e] and backsolve")


# ---------------------------------------------------------------------------------------------------------------------
# 2. the downdate: against the long-double twin per problem
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(33, 20), (129, 129), (2, 1)], ids=lambda s: f"n{s[0]}k{s[1]}")
def test_downdate_ext(D, h, shape):
    n, k = shape
    nrhs, m = 3, n + 5 + k
    fams = finite_families(m, n)
    mats = [F.make(f, m, n) for f in fams]
    Q = cm(D, mats)
    st = D.qr_batched_(Q, handle=h)
    torch.cuda.synchronize()
    R0, a0 = Q.cpu().numpy(), st.α.cpu().numpy()
    rng = np.random.default_rng(n)
    cs = [rng.standard_normal((n, nrhs)) for _ in fams]
    es = [rng.standard_normal((k, nrhs)) for _ in fams]
    Z = cm(D, [a[m - k:] for a in mats])
    c, e = cm(D, cs), cm(D, es)
    t = D.downdate_rows_batched_(Q, st.α, Z, c, e, handle=h)
    torch.cuda.synchronize()
    R1, a1, V2, vt, info, c1, e1 = Q.cpu().numpy(), st.α.cpu().numpy(), t.B.cpu().numpy(), t.vtop.cpu().numpy(), t.info.cpu().numpy(), \
        c.cpu().numpy(), e.cpu().numpy()
    for i, fam in enumerate(fams):
        Rr, ar, Zr = np.asfortranarray(R0[i][:n]), a0[i].copy(), np.asfortranarray(mats[i][m - k:])
        Rm, am, V2m, vtm, infom, cm_, em = M.unblocked(Rr, ar, Zr, cs[i], es[i])
        Re, ae, V2e, vte, infoe, ce, ee = M.ext_downdate(Rr, ar, Zr, cs[i], es[i])
        where = f"{fam} n={n} k={k} problem {i}"
        Rref = full(Re, ae)
        cond = np.abs(full(Rr, ar)).max() / max(np.abs(np.nan_to_num(Rref)).max(), np.finfo(float).tiny)
        if infom or infoe or (info[i] and cond > 1e4):
            continue                                   # impossible in fp64 or long double (test_gpu_downdate.py lists these)
        assert info[i] == 0, f"device info {info[i]} on a removal both references carry out; {where}"
        ref = types.SimpleNamespace(m=n + k, n=n, family=fam)
        Vref = np.vstack([np.diag(vte), V2e])
        gpu = {"R": relerr(full(R1[i], a1[i]), Rref), "V": relerr(np.vstack([np.diag(vt[i]), V2[i]]), Vref),
               "qtb": relerr(np.vstack([c1[i], e1[i]]), np.vstack([ce, ee]))}
        e64 = {"R": relerr(full(Rm, am), Rref), "V": relerr(np.vstack([np.diag(vtm), V2m]), Vref),
               "qtb": relerr(np.vstack([cm_, em]), np.vstack([ce, ee]))}
        DD_TABLE.check(f"downdate_batched n={n} k={k}" + (" (ill-conditioned removal)" if cond > 1e4 else ""), ref, gpu, e64, note=where)


# ---------------------------------------------------------------------------------------------------------------------
# 3. shapes: Gram identities, the single-problem append and applies, the size limit
# ---------------------------------------------------------------------------------------------------------------------
NS = (1, 2, 31, 32, 33, 128, 129, 443, 1000)
KS = ("1", "2", "33", "n", "4n")
NRHS = (0, 1, 3, 65)


def _single_apply(D, h, fn, n, k, V2, vt, c, e):
    """dhqr_apply_qt_append_f64 / dhqr_apply_downdate_f64 on one problem's (V2, vtop)."""
    nrhs = c.shape[1]
    dc, de = D.to_colmajor(c, DEV), D.to_colmajor(e, DEV)
    dV, dv = D.to_colmajor(V2, DEV), torch.from_numpy(vt.copy()).to(DEV)
    D._lib.call(fn, h.raw, n, k, P(dV), k, P(dv), P(dc), n, P(de), k, nrhs, SP(torch.cuda.current_stream()))
    return npy(dc), npy(de)


@pytest.mark.parametrize("nrhs", NRHS)
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("n", NS)
def test_shapes(D, h, n, k, nrhs):
    kk = {"n": n, "4n": 4 * n}.get(k) or int(k)
    ncol = n + nrhs
    nb = 3
    rng = np.random.default_rng([n, kk, nrhs])
    R = [np.triu(rng.standard_normal((n, n)), 1) + np.diag(2.0 + rng.random(n)) * np.sqrt(n) for _ in range(nb)]
    Bs = [rng.standard_normal((kk, n)) for _ in range(nb)]
    cs = [rng.standard_normal((n, nrhs)) for _ in range(nb)]
    es = [rng.standard_normal((kk, nrhs)) for _ in range(nb)]
    dR = cm(D, [np.triu(r, 1) for r in R])
    al = torch.from_numpy(np.stack([np.diag(r) for r in R])).to(DEV).contiguous()
    dB = cm(D, Bs)
    dc, de = (cm(D, cs), cm(D, es)) if nrhs else (None, None)
    if ncol > COLS or kk * ncol > LIM:
        with pytest.raises(ValueError):
            D.append_rows_batched_(dR, al, dB, dc, de, handle=h)
        rc = D._lib.load().dhqr_qr_append_batched_f64(*tp_args(h, n, kk, nb, dR, n, n * n, al, n, dB, kk, kk * n, torch.zeros(nb * n,
                                                               device=DEV, dtype=torch.float64), n, dc, n, n * nrhs, de, kk, kk * nrhs, nrhs), None)
        assert rc == -3
        return
    assert cluster_size(kk, ncol) in (1, 2, 4, 8)
    t = D.append_rows_batched_(dR, al, dB, dc, de, handle=h)
    torch.cuda.synchronize()
    R1, a1, V2, vt = dR.cpu().numpy(), al.cpu().numpy(), t.B.cpu().numpy(), t.vtop.cpu().numpy()
    for i in range(nb):
        Rp = full(R1[i], a1[i])
        G0 = R[i].T @ R[i] + Bs[i].T @ Bs[i]
        assert relerr(Rp.T @ Rp, G0) < 1e-13 * max(8, kk + n) ** 0.5 * 10, (n, kk, nrhs, i)
        # the single-problem append on the same problem
        Ra = D.to_colmajor(np.triu(R[i], 1), DEV)
        aa = torch.from_numpy(np.diag(R[i]).copy()).to(DEV)
        ts = D.append_rows_((Ra, aa), D.to_colmajor(Bs[i], DEV), handle=h)
        assert relerr(Rp, full(npy(Ra), aa.cpu().numpy())) < 1e-12
        if nrhs:
            cref, eref = _single_apply(D, h, "dhqr_apply_qt_append_f64", n, kk, V2[i], vt[i], cs[i], es[i])
            got = np.vstack([dc[i].cpu().numpy(), de[i].cpu().numpy()])
            assert relerr(got, np.vstack([cref, eref])) < 1e-12, (n, kk, nrhs, i)
    # the downdate of the same rows returns to R (up to row signs), its right-hand sides to (c, e)
    dZ = cm(D, Bs)
    dc2, de2 = (cm(D, cs), cm(D, es)) if nrhs else (None, None)
    td = D.downdate_rows_batched_(dR, al, dZ, dc2, de2, handle=h)
    torch.cuda.synchronize()
    info = td.info.cpu().numpy()
    assert (info == 0).all(), info
    R2, a2 = dR.cpu().numpy(), al.cpu().numpy()
    for i in range(nb):
        assert relerr(signed(full(R2[i], a2[i])), signed(R[i])) < 1e-10 * max(1, kk / n), (n, kk, nrhs, i)
        if nrhs:
            cref, eref = _single_apply(D, h, "dhqr_apply_downdate_f64", n, kk, td.B[i].cpu().numpy(), td.vtop[i].cpu().numpy(), cs[i], es[i])
            got = np.vstack([dc2[i].cpu().numpy(), de2[i].cpu().numpy()])
            assert relerr(got, np.vstack([cref, eref])) < 1e-10, (n, kk, nrhs, i)


def test_size_limit(D, h):
    """Exactly at the limits the calls run; one row or one column past them they are refused with -3 before any launch."""
    lib = D._lib.load()
    assert h.get_option("batch_update_max_cols") == COLS and h.get_option("batch_max_elems") == LIM
    for n, nrhs in ((1000, 24), (4, 0), (64, 1)):
        ncol = n + nrhs
        k = LIM // ncol
        assert cluster_size(k, ncol) == 8 or k * ncol <= SLAB
        R = torch.zeros(n * n, dtype=torch.float64, device=DEV)
        al = torch.ones(n, dtype=torch.float64, device=DEV)
        B = torch.randn(k * n + n * ncol, dtype=torch.float64, device=DEV)
        vt = torch.zeros(n, dtype=torch.float64, device=DEV)
        c = torch.zeros(max(n * nrhs, 1), dtype=torch.float64, device=DEV)
        e = torch.randn(max((k + 1) * nrhs, 1), dtype=torch.float64, device=DEV)
        cc, ee = (c, e) if nrhs else (None, None)
        B0 = B.clone()                                  # B is overwritten with the reflector tails
        l0 = h.launch_count()
        assert lib.dhqr_qr_append_batched_f64(*tp_args(h, n, k, 1, R, n, 0, al, 0, B, k, 0, vt, 0, cc, n, 0, ee, k, 0, nrhs), None) == 0
        torch.cuda.synchronize()
        assert h.launch_count() == l0 + 1 and torch.isfinite(al).all()
        Rp = torch.triu(R.view(n, n).T, 1) + torch.diag(al)
        G = B0[:k * n].view(n, k) @ B0[:k * n].view(n, k).T + torch.eye(n, dtype=torch.float64, device=DEV)
        assert ((Rp.T @ Rp - G).abs().max() / G.abs().max()).item() < 1e-12
        l0 = h.launch_count()
        assert lib.dhqr_qr_append_batched_f64(*tp_args(h, n, k + 1, 1, R, n, 0, al, 0, B, k + 1, 0, vt, 0, cc, n, 0, ee, k + 1, 0, nrhs),
                                              None) == -3
        assert h.launch_count() == l0
    x = torch.zeros(4 * 1025 * 1025, dtype=torch.float64, device=DEV)
    assert lib.dhqr_qr_append_batched_f64(*tp_args(h, 1000, 1, 1, x, 1000, 0, x[-2000:], 0, x[1001000:], 1, 0, x[-1000:], 0, x[2002000:],
                                                   1000, 0, x[2100000:], 1, 0, 25), None) == -3
    assert lib.dhqr_backsolve_batched_f64(h.raw, 1025, 1, P(x), 1025, 0, P(x[-2000:]), 0, P(x[2000000:]), 1025, 0, 1, None) == -2
    assert lib.dhqr_backsolve_batched_f64(h.raw, 1024, 1, P(x), 1024, 0, P(x[-2000:]), 0, P(x[2000000:]), 1024, 0, 1, None) == 0


def test_from_zero(D, h):
    """From R = 0 (alpha = 0) the append gives R'R' = B'B."""
    nb, n, k = 4, 40, 100
    B0 = torch.randn(nb, k, n, dtype=torch.float64, device=DEV)
    R = D.colmajor_empty_batched(nb, n, n, DEV)
    R.zero_()
    al = torch.zeros(nb, n, dtype=torch.float64, device=DEV)
    B = D.colmajor_empty_batched(nb, k, n, DEV)
    B.copy_(B0)
    D.append_rows_batched_(R, al, B, handle=h)
    Rp = torch.triu(R, 1) + torch.diag_embed(al)
    G = B0.transpose(1, 2) @ B0
    assert ((Rp.transpose(1, 2) @ Rp - G).abs().amax((1, 2)) / G.abs().amax((1, 2))).max().item() < 1e-13


# ---------------------------------------------------------------------------------------------------------------------
# 4. failure: one problem removes rows it never had
# ---------------------------------------------------------------------------------------------------------------------
def test_failure_isolated(D, h):
    nb, n, k, nrhs, bad = 5, 24, 6, 2, 2
    g = torch.Generator(device=DEV).manual_seed(4)
    A = torch.randn(nb, 60, n, dtype=torch.float64, device=DEV, generator=g)
    Z = torch.randn(nb, k, n, dtype=torch.float64, device=DEV, generator=g)
    Z[:, :, :] = A[:, :k]
    Z[bad] = 100.0 * torch.randn(k, n, dtype=torch.float64, device=DEV, generator=g)     # never added
    c0 = torch.randn(nb, n, nrhs, dtype=torch.float64, device=DEV, generator=g)
    e0 = torch.randn(nb, k, nrhs, dtype=torch.float64, device=DEV, generator=g)

    def run(idx):
        Q = cm(D, [A[i].cpu().numpy() for i in idx])
        st = D.qr_batched_(Q, handle=h)
        Zb, c, e = cm(D, [Z[i].cpu().numpy() for i in idx]), cm(D, [c0[i].cpu().numpy() for i in idx]), cm(D, [e0[i].cpu().numpy() for i in idx])
        t = D.downdate_rows_batched_(Q, st.α, Zb, c, e, handle=h)
        torch.cuda.synchronize()
        return Q, st.α, t.B, t.vtop, t.info, c, e

    full_ = run(list(range(nb)))
    rest = [i for i in range(nb) if i != bad]
    part = run(rest)
    info = full_[4].cpu().numpy()
    assert info[bad] >= 1 and (np.delete(info, bad) == 0).all(), info
    j = int(info[bad]) - 1
    al = full_[1][bad].cpu().numpy()
    assert np.isnan(al[j:]).all() and np.isfinite(al[:j]).all()
    assert (full_[3][bad, j:] == 0).all() and (full_[2][bad, :, j:] == 0).all()
    for p, i in enumerate(rest):
        for x, y in zip(full_, part):
            if x.dim() == 1:
                continue
            assert same_bits(x[i], y[p]), f"problem {i}"


# ---------------------------------------------------------------------------------------------------------------------
# 5. the batched back-substitution on qr_batched_ factors, by the rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(40, 33), (300, 129), (2, 1)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_backsolve_ext(D, h, coracle, oracle, shape):
    m, n = shape
    nrhs = 3
    refs = [E.Ref(coracle, oracle, f, m, n, nrhs=nrhs) for f in finite_families(m, n)]
    refs = [r for r in refs if r.solve]
    Q = cm(D, [r.A for r in refs])
    st = D.qr_batched_(Q, handle=h)
    b = cm(D, [r.b for r in refs])
    D.apply_qt_batched_(b, Q, h)
    Rn = poisoned(D, Q, n)
    keep = b[:, n:].clone()
    D.backsolve_batched_(b, Rn, st.α, h)
    torch.cuda.synchronize()
    assert same_bits(b[:, n:], keep)
    x = b[:, :n].cpu().numpy()
    for i, ref in enumerate(refs):
        g = {"x": E.nrm(x[i] - ref.x_e) / E.nrm(ref.x_e)}
        e64 = {"x": E.nrm(ref.x64 - ref.x_e) / E.nrm(ref.x_e)}
        TABLE.check(f"backsolve_batched {m}x{n}", ref, g, e64, note=f"problem {i}, block of {nrhs} right-hand sides")


# ---------------------------------------------------------------------------------------------------------------------
# 6. the rolling solver
# ---------------------------------------------------------------------------------------------------------------------
def test_rolling_solver(D, h):
    nb, n, w, step, slides = 300, 16, 200, 10, 50
    g = torch.Generator(device=DEV).manual_seed(21)
    T = w + step * slides
    A = torch.randn(nb, T, n, dtype=torch.float64, device=DEV, generator=g)
    xt = torch.randn(nb, n, 1, dtype=torch.float64, device=DEV, generator=g)
    b = (A @ xt)[..., 0] + 0.1 * torch.randn(nb, T, dtype=torch.float64, device=DEV, generator=g)
    ls = D.BatchedStreamingLeastSquares(nb, n, handle=h)
    ls.add(A[:, :w], b[:, :w])
    worst_x = worst_r = 0.0
    for s in range(slides):
        lo, hi = s * step, w + s * step
        l0 = h.launch_count()
        ls.add(A[:, hi:hi + step], b[:, hi:hi + step])
        info = ls.remove(A[:, lo:lo + step], b[:, lo:lo + step])
        x = ls.solve()
        assert h.launch_count() == l0 + 3
        Aw, bw = A[:, lo + step:hi + step], b[:, lo + step:hi + step]
        xl = torch.linalg.lstsq(Aw, bw[..., None]).solution[..., 0]
        worst_x = max(worst_x, ((x - xl).norm(dim=1) / xl.norm(dim=1)).max().item())
        rd = (Aw @ xl[..., None])[..., 0].sub(bw).norm(dim=1)
        worst_r = max(worst_r, ((ls.residual_norm() - rd).abs() / rd).max().item())
        assert (info == 0).all()
    assert (ls.rows == w).all()
    assert worst_x < 1e-11 and worst_r < 1e-9, (worst_x, worst_r)
    # a failed removal leaves that problem as it was; the others are downdated
    before = (ls.A.clone(), ls.α.clone(), ls.c.clone(), ls._ss.clone(), ls.rows.clone())
    Zb, eb = A[:, T - w:T - w + step].clone(), b[:, T - w:T - w + step].clone()
    Zb[7] = 50.0 * torch.randn(step, n, dtype=torch.float64, device=DEV, generator=g)
    info = ls.remove(Zb, eb).cpu().numpy()
    assert info[7] > 0 and (np.delete(info, 7) == 0).all()
    after = (ls.A, ls.α, ls.c, ls._ss, ls.rows)
    for x0, x1 in zip(before, after):
        assert same_bits(x0[7:8], x1[7:8])
    assert int(ls.rows[0]) == w - step and int(ls.rows[7]) == w


# ---------------------------------------------------------------------------------------------------------------------
# 7. contracts
# ---------------------------------------------------------------------------------------------------------------------
def layout_run(D, h, R0, a0, B0, c0, e0, hyp, order, lds=(0, 0, 0, 0), gaps=(0, 0, 0, 0, 0, 0), off=0):
    """One call on the problems `order` of (R0, a0, B0, c0, e0) in NaN-fenced buffers with extra leading dimensions, stride gaps and
    an 8 B base offset; returns the outputs per problem in `order` and whether every sentinel survived."""
    lib = D._lib.load()
    nb = len(order)
    _, n, _ = R0.shape
    k, nrhs = B0.shape[1], c0.shape[2]
    ldr, ldb, ldc, lde = n + lds[0], k + lds[1], n + lds[2], k + lds[3]
    sr, sal, sb, svt, sc, se = ldr * n + gaps[0], n + gaps[1], ldb * n + gaps[2], n + gaps[3], ldc * nrhs + gaps[4], lde * nrhs + gaps[5]
    bufs = {}

    def fenced(name, stride, shape, strides, src):
        base = torch.full((off + nb * stride + 7,), float("nan"), dtype=torch.float64, device=DEV)
        v = base[off:off + nb * stride].as_strided(shape, strides)
        for p, i in enumerate(order):
            v[p].copy_(src[i])
        bufs[name] = (base, v)
        return v
    iu = torch.triu(torch.ones(n, n, dtype=torch.bool, device=DEV), 1)
    R = fenced("R", sr, (nb, n, n), (sr, 1, ldr), torch.where(iu, R0, torch.full_like(R0, float("nan"))))
    al = fenced("al", sal, (nb, n), (sal, 1), a0)
    B = fenced("B", sb, (nb, k, n), (sb, 1, ldb), B0)
    vt = fenced("vt", svt, (nb, n), (svt, 1), torch.zeros(len(a0), n, dtype=torch.float64, device=DEV))
    c = fenced("c", sc, (nb, n, nrhs), (sc, 1, ldc), c0)
    e = fenced("e", se, (nb, k, nrhs), (se, 1, lde), e0)
    info = torch.full((nb + 2,), -7, dtype=torch.int64, device=DEV)
    keep = {name: bb.clone() for name, (bb, _) in bufs.items()}
    fn = lib.dhqr_qr_downdate_batched_f64 if hyp else lib.dhqr_qr_append_batched_f64
    args = tp_args(h, n, k, nb, C.c_void_p(R.data_ptr()), ldr, sr, C.c_void_p(al.data_ptr()), sal, C.c_void_p(B.data_ptr()), ldb, sb,
                   C.c_void_p(vt.data_ptr()), svt, C.c_void_p(c.data_ptr()), ldc, sc, C.c_void_p(e.data_ptr()), lde, se, nrhs)
    if hyp:
        args.append(C.c_void_p(info.data_ptr() + 8))
    assert fn(*args, SP(torch.cuda.current_stream())) == 0
    torch.cuda.synchronize()
    ok = True
    for name, (base, v) in bufs.items():
        mask = torch.ones_like(base, dtype=torch.bool)
        idx = torch.arange(base.numel(), device=DEV)
        mask[idx[off:].as_strided(v.shape, v.stride()).flatten()] = False
        # R: only the strict upper triangle is written; its diagonal and lower part keep the caller's data
        ok = ok and bool(same_bits(base[mask], keep[name][mask]))
    ok = ok and int(info[0]) == -7 and int(info[-1]) == -7
    outs = [(torch.triu(R[p], 1), al[p], B[p], vt[p], c[p], e[p]) + ((info[1 + p:2 + p],) if hyp else ()) for p in range(nb)]
    return outs, ok, R


def contract_data(nb=5, n=33, k=40, nrhs=3, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = torch.randn(nb, 2 * n + k, n, dtype=torch.float64, device=DEV, generator=g)
    Rq = torch.linalg.qr(A[:, :n + k]).R
    sg = torch.sign(torch.diagonal(Rq, dim1=1, dim2=2))
    Rq = Rq * sg[..., None]
    R0 = torch.triu(Rq, 1)
    a0 = torch.diagonal(Rq, dim1=1, dim2=2).contiguous()
    B0 = A[:, n:n + k].contiguous()               # rows of the factored block: removable, and a fine block to append
    c0 = torch.randn(nb, n, nrhs, dtype=torch.float64, device=DEV, generator=g)
    e0 = torch.randn(nb, k, nrhs, dtype=torch.float64, device=DEV, generator=g)
    return R0, a0, B0, c0, e0


@pytest.mark.parametrize("hyp", [False, True], ids=["append", "downdate"])
def test_bitwise_layout(D, h, hyp):
    data = contract_data()
    nb = data[0].shape[0]
    ref = [layout_run(D, h, *data, hyp, [i])[0][0] for i in range(nb)]
    order = list(range(nb))[::-1]
    for off in (0, 1):
        outs, ok, R = layout_run(D, h, *data, hyp, order, lds=(3, 5, 2, 7), gaps=(7, 2, 3, 1, 5, 4), off=off)
        assert ok, f"a sentinel changed (offset {off})"
        assert torch.isnan(R[:, ~torch.triu(torch.ones(R.shape[1], R.shape[2], dtype=torch.bool, device=DEV), 1)]).all(), \
            "R's diagonal or lower part was written"
        for p, i in enumerate(order):
            for x, y in zip(outs[p], ref[i]):
                assert same_bits(x, y), f"problem {i}, offset {off}"
    two = layout_run(D, h, *data, hyp, [3, 1])[0]
    for p, i in enumerate([3, 1]):
        for x, y in zip(two[p], ref[i]):
            assert same_bits(x, y)


def test_large_batch(D, h):
    """B spans more than 2^31 bytes: a seeded sample of positions equals batch = 1 calls."""
    n, k, nb = 4, 64, (1 << 31) // (8 * 4 * 64) + 3
    g = torch.Generator(device=DEV).manual_seed(9)
    B = D.colmajor_empty_batched(nb, k, n, DEV)
    B.copy_(torch.randn(nb, n, k, dtype=torch.float64, device=DEV, generator=g).transpose(1, 2))
    assert B.numel() * 8 > 2 ** 31
    R = D.colmajor_empty_batched(nb, n, n, DEV)
    R.copy_(torch.randn(nb, n, n, dtype=torch.float64, device=DEV, generator=g))
    al = torch.rand(nb, n, dtype=torch.float64, device=DEV, generator=g) + 1.0
    pos = sorted(set(np.random.default_rng(3).integers(0, nb, 12).tolist()) | {0, nb - 1})
    src = {p: (R[p].clone(), al[p].clone(), B[p].clone()) for p in pos}
    t = D.append_rows_batched_(R, al, B, handle=h)
    for p in pos:
        R1, a1, B1 = cm(D, [src[p][0].cpu().numpy()]), src[p][1][None].clone(), cm(D, [src[p][2].cpu().numpy()])
        t1 = D.append_rows_batched_(R1, a1, B1, handle=h)
        assert same_bits(R[p], R1[0]) and same_bits(al[p], a1[0]) and same_bits(t.B[p], t1.B[0]) and same_bits(t.vtop[p], t1.vtop[0]), p
    del B, R


CN, CK, CB, CR = 32, 48, 200, 2


def contract_calls(lib, hraw, bufs, s):
    R, al, B, vt, c, e, Z, vz, c2, e2, info, b = bufs
    return {"append": lambda: lib.dhqr_qr_append_batched_f64(hraw, CN, CK, CB, P(R), CN, CN * CN, P(al), CN, P(B), CK, CK * CN, P(vt), CN,
                                                             P(c), CN, CN * CR, P(e), CK, CK * CR, CR, s),
            "downdate": lambda: lib.dhqr_qr_downdate_batched_f64(hraw, CN, CK, CB, P(R), CN, CN * CN, P(al), CN, P(Z), CK, CK * CN, P(vz),
                                                                 CN, P(c2), CN, CN * CR, P(e2), CK, CK * CR, CR, P(info), s),
            "backsolve": lambda: lib.dhqr_backsolve_batched_f64(hraw, CN, CB, P(R), CN, CN * CN, P(al), CN, P(b), CN, CN * CR, CR, s)}


def contract_bufs(D, seed=0):
    R0, a0, B0, c0, e0 = contract_data(CB, CN, CK, CR, seed)
    R = cm(D, list(R0.cpu().numpy()))
    return [R, a0.clone(), cm(D, list(B0.cpu().numpy())), torch.zeros(CB, CN, dtype=torch.float64, device=DEV), cm(D, list(c0.cpu().numpy())),
            cm(D, list(e0.cpu().numpy())), cm(D, list(B0.cpu().numpy())), torch.zeros(CB, CN, dtype=torch.float64, device=DEV),
            cm(D, list(c0.cpu().numpy())), cm(D, list(e0.cpu().numpy())), torch.zeros(CB, dtype=torch.int64, device=DEV),
            cm(D, list(c0.cpu().numpy()))]


def run_contract(D, hd, name, s=None):
    bufs = contract_bufs(D)
    lib = D._lib.load()
    torch.cuda.synchronize()
    assert contract_calls(lib, hd.raw, bufs, SP(s or torch.cuda.current_stream()))[name]() == 0
    torch.cuda.synchronize()
    return bufs


@pytest.mark.parametrize("name", ["append", "downdate", "backsolve"])
def test_gated_side_stream(D, h, name):
    ref = run_contract(D, h, name)
    g = Gate()
    s = torch.cuda.Stream()
    bufs = contract_bufs(D)
    keep = [x.clone() for x in bufs]
    for x in bufs:
        x.fill_(float("nan")) if x.dtype == torch.float64 else x.fill_(-1)
    torch.cuda.synchronize()
    ev = g.close(s)
    with torch.cuda.stream(s):
        for x, y in zip(bufs, keep):
            x.copy_(y)
        rc = contract_calls(D._lib.load(), h.raw, bufs, SP(s))[name]()
    closed = not ev.query()
    assert rc == 0 and closed, f"{name} blocked the host until the caller's stream drained"
    torch.cuda.synchronize()
    assert all(same_bits(x, y) for x, y in zip(bufs, ref)), name


def test_graph_capture_fresh_handle(D):
    h2 = D.Handle(0)
    try:
        ref = {name: run_contract(D, h2, name) for name in ("append", "downdate", "backsolve")}
        h3 = D.Handle(0)
        try:
            bufs = contract_bufs(D)
            keep = [x.clone() for x in bufs]
            lib = D._lib.load()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, capture_error_mode="global"):
                calls = contract_calls(lib, h3.raw, bufs, SP(torch.cuda.current_stream()))
                for name in ("append", "downdate", "backsolve"):
                    assert calls[name]() == 0
            for x, y in zip(bufs, keep):
                x.copy_(y)
            gr.replay()
            torch.cuda.synchronize()
            # append then downdate of the same rows, then the backsolve on the result: compare with the three calls in sequence
            seq = contract_bufs(D)
            calls = contract_calls(lib, h2.raw, seq, SP(torch.cuda.current_stream()))
            for name in ("append", "downdate", "backsolve"):
                assert calls[name]() == 0
            torch.cuda.synchronize()
            assert all(same_bits(x, y) for x, y in zip(bufs, seq))
            for name in ref:                        # and each call on a fresh handle gives the bits of any other
                assert all(same_bits(x, y) for x, y in zip(ref[name], run_contract(D, h3, name))), name
        finally:
            torch.cuda.synchronize()
            h3.close()
    finally:
        h2.close()


def test_history_and_launch_count(D):
    h2 = D.Handle(0)
    try:
        first = {name: run_contract(D, h2, name) for name in ("append", "downdate", "backsolve")}
        M_ = D.colmajor_empty(2000, 300, DEV)
        D.fill_uniform_(M_, 3, handle=h2)
        st = D.qr_(M_, handle=h2)
        D.ldiv(st, torch.ones(2000, dtype=torch.float64, device=DEV))
        big = D.colmajor_empty_batched(400, 4096, 48, DEV)
        big.normal_()
        D.qr_batched_(big, handle=h2)
        ls = D.BatchedStreamingLeastSquares(50, 100, nrhs=3, handle=h2)
        ls.add(torch.randn(50, 1500, 100, dtype=torch.float64, device=DEV), torch.randn(50, 1500, 3, dtype=torch.float64, device=DEV))
        ls.solve()
        torch.cuda.synchronize()
        for name in first:
            l0 = h2.launch_count()
            again = run_contract(D, h2, name)
            assert h2.launch_count() == l0 + 1, name
            assert all(same_bits(x, y) for x, y in zip(first[name], again)), name
        with E.options(h2, profile=1):
            bufs = contract_bufs(D)
            for fn in contract_calls(D._lib.load(), h2.raw, bufs, SP(torch.cuda.current_stream())).values():
                assert fn() == 0
            prof = h2.profile()
            for cls in ("k_append_batched", "k_downdate_batched", "k_backsolve_batched"):
                assert prof[cls]["count"] == 1, (cls, prof)
    finally:
        torch.cuda.synchronize()
        h2.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors(D, h):
    lib = D._lib.load()
    n, k, nb, r = 4, 6, 3, 2
    sizes = [nb * n * n, nb * n, nb * k * n, nb * n, nb * n * r, nb * k * r, nb]
    offs = np.cumsum([0] + sizes)
    buf = torch.zeros(int(offs[-1]) + 64, dtype=torch.float64, device=DEV)
    ptr = [C.c_void_p(buf.data_ptr() + 8 * int(o)) for o in offs[:-1]]
    R, al, B, vt, c, e, info = ptr
    mis = C.c_void_p(buf.data_ptr() + 4)
    s = SP(torch.cuda.current_stream())
    ap = [h.raw, n, k, nb, R, n, n * n, al, n, B, k, k * n, vt, n, c, n, n * r, e, k, k * r, r, s]
    dd = ap[:-1] + [info, s]
    bs = [h.raw, n, nb, R, n, n * n, al, n, c, n, n * r, r, s]
    common = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, LIM), (1, 1025)], -4: [(3, -1), (3, 2 ** 31)],
              -5: [(4, None), (4, mis)], -6: [(5, n - 1)], -7: [(6, n * n - 1)], -8: [(7, None), (7, mis), (7, R)], -9: [(8, n - 1)],
              -10: [(9, None), (9, mis), (9, R), (9, al)], -11: [(10, k - 1)], -12: [(11, k * n - 1)],
              -13: [(12, None), (12, mis), (12, R), (12, al), (12, B)], -14: [(13, n - 1)],
              -15: [(14, None), (14, mis), (14, R), (14, al), (14, B), (14, vt)], -16: [(15, n - 1)], -17: [(16, n * r - 1)],
              -18: [(17, None), (17, mis), (17, R), (17, al), (17, B), (17, vt), (17, c)], -19: [(18, k - 1)], -20: [(19, k * r - 1)],
              -21: [(20, -1)]}
    table = {
        "dhqr_qr_append_batched_f64": (ap, common),
        "dhqr_qr_downdate_batched_f64": (dd, {**common, -22: [(21, None), (21, mis), (21, R), (21, al), (21, B), (21, vt), (21, c), (21, e)]}),
        "dhqr_backsolve_batched_f64": (bs, {-1: [(0, None)], -2: [(1, -1), (1, 1025)], -3: [(2, -1), (2, 2 ** 31)], -4: [(3, None), (3, mis)],
                                            -5: [(4, n - 1)], -6: [(5, n * n - 1)], -7: [(6, None), (6, mis)], -8: [(7, n - 1)],
                                            -9: [(8, None), (8, mis), (8, R), (8, al)], -10: [(9, n - 1)], -11: [(10, n * r - 1)],
                                            -12: [(11, -1)]}),
    }
    keep = buf.clone()
    torch.cuda.synchronize()
    l0 = h.launch_count()
    for fn, (args, cases) in table.items():
        f = getattr(lib, fn)
        for code, subs in cases.items():
            for idx, val in subs:
                a = list(args)
                a[idx] = val
                assert f(*a) == code, (fn, code, idx, val, lib.dhqr_last_error())
        noops = (3, 1, 2) if fn != "dhqr_backsolve_batched_f64" else (2, 1, 11)
        for idx in noops:                           # batch = 0, n = 0, k = 0 (nrhs = 0 for the backsolve)
            a = list(args)
            a[idx] = 0
            assert f(*a) == 0, (fn, idx)
    # nrhs = 0 with null c and e runs (and transforms nothing)
    a = list(ap)
    a[14], a[17], a[20] = None, None, 0
    assert same_bits(buf, keep) and h.launch_count() == l0
    assert lib.dhqr_qr_append_batched_f64(*a) == 0
    assert h.launch_count() == l0 + 1
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="batch_update_max_cols"):
        D.BatchedStreamingLeastSquares(2, 1024, handle=h)


def _multi_rank_job(rank, P_, _marker):
    import dhqr_b200 as D2
    h2 = D2.init_distributed(device=0)
    lib = D2._lib.load()
    x = torch.zeros(512, dtype=torch.float64, device=DEV)
    p = [C.c_void_p(x.data_ptr() + 8 * 64 * i) for i in range(8)]
    l0 = h2.launch_count()
    codes = [lib.dhqr_qr_append_batched_f64(h2.raw, 4, 4, 1, p[0], 4, 16, p[1], 4, p[2], 4, 16, p[3], 4, p[4], 4, 4, p[5], 4, 4, 1, None),
             lib.dhqr_qr_downdate_batched_f64(h2.raw, 4, 4, 1, p[0], 4, 16, p[1], 4, p[2], 4, 16, p[3], 4, p[4], 4, 4, p[5], 4, 4, 1, p[6],
                                              None),
             lib.dhqr_backsolve_batched_f64(h2.raw, 4, 1, p[0], 4, 16, p[1], 4, p[4], 4, 4, 1, None)]
    out = {"codes": np.array(codes), "launches": np.array(h2.launch_count() - l0)}
    D2.shutdown_distributed()
    return out


L.JOBS.setdefault("batched_update_multi_rank", _multi_rank_job)


def test_multi_rank_handle(tmp_path):
    d, so = L.build()
    try:
        ranks = L.run(2, "batched_update_multi_rank", str(tmp_path), so, args=(_multi_rank_job,))
    except L.Skip as e:
        pytest.skip(f"the loopback transport cannot run here: {e}")
    finally:
        shutil.rmtree(d, ignore_errors=True)
    for r, res in enumerate(ranks):
        assert res["codes"].tolist() == [-1, -1, -1] and int(res["launches"]) == 0, f"rank {r}"
