"""Deleting rows from a factorisation on the device (dhqr_qr_downdate_f64, dhqr_apply_downdate_f64; DESIGN §2.11), and sliding-window
least squares (StreamingLeastSquares.remove).

Accuracy: R', vtop and V2 are held to the extended-precision rule of ext_rule.py against the long-double twin of the unblocked
recurrence (tests/downdate_ext.c) run on the device's own R, with the fp64 blocked model (tests/downdate_model.py) as the fp64
oracle; the ratio table goes to build/downdate_ext.md.  On top: R' against the long-double R of the remaining rows, least squares
on the remaining rows, a sliding window, the failure rule, and the storage, stream, launch-accounting, memory and argument
contracts.

The module also registers qr_downdate and apply_downdate in test_gpu_history.py's catalogue at import, so every history there
covers the new entry points.  The catalogue check (test_catalogue_covers_the_header) therefore needs tests/ collected as a whole
(pytest tests ...): this module sorts before test_gpu_history.py and is imported first."""
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
from test_gpu_streams import P, SP, Case, dev, gate, run_gated, same_bits  # noqa: F401  (gate: the fixture)

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
FAMILIES = tuple(f for f in F.FAMILIES if f not in F.NAN_FAMILIES)
NS = (1, 31, 32, 33, 127, 128, 129, 500, 1024)
KS = ("1", "2", "31", "33", "255", "n")
ILL = 1e4                      # ||R|| / ||R'|| above this: the removal itself is ill-conditioned (reported as such in the table)


class Table(E.Table):
    """The ratio table, plus one line per cell whose removal the fp64 recurrence (model or long double) found impossible."""

    def __init__(self, name):
        super().__init__(name)
        self.notes = []

    def write(self):
        super().write()
        if self.notes:
            import os
            path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", self.name)
            try:
                with open(path, "a") as fh:
                    fh.write("\nnot held to the rule (the removal is impossible in fp64 or long double at this shape):\n\n")
                    fh.write("\n".join(f"- {n}" for n in self.notes) + "\n")
            except OSError:
                pass


TABLE = Table("downdate_ext.md")


# ---------------------------------------------------------------------------------------------------------------------
# the history catalogue: the downdate of the catalogue's own factorisation (X["H"], the qr of X["A"]) by its first KD rows
# ---------------------------------------------------------------------------------------------------------------------
KD = 200


@HIST.case("qr_downdate", "dhqr_qr_downdate_f64")
def _hist_downdate(h, s, X):
    R, al, Z, vt = HIST.up(X["H"]), HIST.up(X["alpha"]), HIST.up(np.asfortranarray(X["A"][:KD])), HIST.zeros(HIST.N)
    info = HIST.zeros(1, torch.int64)
    HIST.call("dhqr_qr_downdate_f64", h.raw, HIST.N, KD, HIST.P(R), HIST.M, HIST.P(al), HIST.P(Z), KD, HIST.P(vt), HIST.P(info),
              HIST.SP(s))
    return {"R": R, "alpha": al, "Z": Z, "vtop": vt, "info": info}


@HIST.case("apply_downdate_r3", "dhqr_apply_downdate_f64")
def _hist_apply(h, s, X):
    if "dd_V2" not in X:                 # the reflectors, once, from a downdate on a handle of their own
        hd, sd = D_().Handle(0), torch.cuda.Stream()
        try:
            with torch.cuda.stream(sd):
                o = _hist_downdate(hd, sd, X)
            sd.synchronize()
            X["dd_V2"], X["dd_vtop"] = o["Z"].cpu().numpy(), o["vtop"].cpu().numpy()
        finally:
            hd.close()
    Z, vt, c, e = HIST.up(X["dd_V2"]), HIST.up(X["dd_vtop"]), HIST.up(X["ca"]), HIST.up(np.asfortranarray(X["ea"][:KD]))
    HIST.call("dhqr_apply_downdate_f64", h.raw, HIST.N, KD, HIST.P(Z), KD, HIST.P(vt), HIST.P(c), HIST.N, HIST.P(e), KD, 3, HIST.SP(s))
    return {"c": c, "e": e}


def D_():
    import dhqr_b200
    return dhqr_b200


# ---------------------------------------------------------------------------------------------------------------------
# fixtures and helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def D():
    return D_()


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


def kval(k, n):
    return n if k == "n" else int(k)


def start(D, h, family, n, k, nb=0, seed=0):
    """The library's factorisation of n + 5 + k rows of a family matrix; the rows to remove (Z) are its last k rows."""
    A = F.make(family, n + 5 + k, n, seed=seed)
    with E.options(h, wide_panel=0):
        dA = D.to_colmajor(A, DEV)
        st = D.qr_(dA, nb=nb, handle=h)
        torch.cuda.synchronize()
    return st, A


def downdate(D, h, st, Z):
    dZ = D.to_colmajor(Z, DEV)
    t = D.downdate_rows_(st, dZ, handle=h)
    torch.cuda.synchronize()
    return t


def full(R, alpha):
    n = alpha.size
    return np.triu(R[:n, :n], 1) + np.diag(alpha)


def signed(R):
    d = np.sign(np.diag(R))
    d[d == 0] = 1.0
    return d[:, None] * R


def sb(a, b):
    """same_bits on any layout."""
    return same_bits(a.contiguous(), b.contiguous())


def relerr(got, ref):
    s = np.abs(ref).max()
    return float(np.abs(got - ref).max() / s) if s > 0 else float(np.abs(got).max())


# ---------------------------------------------------------------------------------------------------------------------
# accuracy: the extended-precision rule against the long-double twin on the device's own R
# ---------------------------------------------------------------------------------------------------------------------
def check_ext(D, h, family, n, k, nb, path):
    st, A = start(D, h, family, n, k, nb)
    R0, a0 = npy(st.A)[:n, :n].copy(), st.α.cpu().numpy().copy()
    Z = np.asfortranarray(A[n + 5:])
    t = downdate(D, h, st, Z)
    info = int(t.info.item())
    Rg, ag, V2g, vtg = npy(st.A)[:n, :n], st.α.cpu().numpy(), npy(t.B), t.vtop.cpu().numpy()
    Rm, am, V2m, vtm, infom = M.qr_downdate(R0, a0, Z)
    Re, ae, V2e, vte, infoe = M.ext_downdate(np.asfortranarray(R0), a0, Z)
    where = f"{path} {family} n={n} k={k}"
    Rref = full(Re, ae)
    cond = np.abs(full(R0, a0)).max() / max(np.abs(np.nan_to_num(Rref)).max(), np.finfo(float).tiny)
    if infom or infoe or (info and cond > ILL):
        TABLE.notes.append(f"{where}: info fp64 model {infom}, long double {infoe}, device {info}; ||R||/||R'|| {cond:.1e}")
        return
    assert info == 0, f"device info {info} on a removal both references carry out; {where}"
    ref = types.SimpleNamespace(m=n + k, n=n, family=family)
    Vref = np.vstack([np.diag(vte), V2e])
    gpu = {"R": relerr(full(Rg, ag), Rref), "V": relerr(np.vstack([np.diag(vtg), V2g]), Vref)}
    e64 = {"R": relerr(full(Rm, am), Rref), "V": relerr(np.vstack([np.diag(vtm), V2m]), Vref)}
    TABLE.check(path + (" (ill-conditioned removal)" if cond > ILL else ""), ref, gpu, e64, note=where)


@pytest.mark.parametrize("family", FAMILIES)
def test_ext_families(D, h, family):
    for n, k in ((129, 33), (256, 255)):
        check_ext(D, h, family, n, k, 0, "downdate nb=0")


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("k", KS)
def test_ext_shapes(D, h, n, k):
    check_ext(D, h, "normal", n, kval(k, n), 0, "downdate shapes")


@pytest.mark.parametrize("nb", (64, 1))
@pytest.mark.parametrize("family", ("graded6", "colscale", "kahan", "normal"))
def test_ext_from_other_paths(D, h, nb, family):
    check_ext(D, h, family, 200, 90, nb, f"downdate after nb={nb}")


@pytest.mark.parametrize("family", ("normal", "uniform", "centered"))
@pytest.mark.parametrize("n,k", ((200, 90), (300, 700)))
def test_against_remaining_rows(D, h, coracle, family, n, k):
    """R' against the long-double R of the rows that remain, up to row signs: no further from it than 8 x the fp64 model's
    downdate of the same R (the hyperbolic form's own error grows with ||R|| / ||R'||), or the floor."""
    st, A = start(D, h, family, n, k)
    R0, a0 = npy(st.A)[:n, :n].copy(), st.α.cpu().numpy().copy()
    Z = np.asfortranarray(A[n + 5:])
    downdate(D, h, st, Z)
    He, ae = coracle.qr_ext(np.asfortranarray(A[:n + 5]))
    Rref = signed(full(He, ae))
    got = relerr(signed(full(npy(st.A), st.α.cpu().numpy())), Rref)
    Rm, am = M.qr_downdate(R0, a0, Z)[:2]
    e64 = relerr(signed(full(Rm, am)), Rref)
    assert got <= E.C_REL * max(e64, E.FLOOR_EPS * E.EPS), (got, e64)


@pytest.mark.parametrize("family", ("normal", "centered", "colscale"))
@pytest.mark.parametrize("m0,n,k", ((400, 128, 77), (2200, 200, 1500)))
def test_lstsq_after_downdate(D, h, coracle, family, m0, n, k):
    """x' = R'^{-1} c' and the residual norm against the long-double solution on the remaining m0 rows."""
    A = F.make(family, m0 + k, n, seed=7)
    b = F.rhs(m0 + k, 2, seed=5).reshape(m0 + k, 2, order="F")
    Ar, br = np.asfortranarray(A[:m0]), np.asfortranarray(b[:m0])
    x_e = coracle.ldiv_ext(Ar, br)
    H64, a64 = coracle.qr(Ar.copy(order="F"))
    x64 = np.stack([coracle.ldiv(H64, a64, br[:, r].copy()) for r in range(2)], 1)
    ls = D.StreamingLeastSquares(n, 2, device=0, handle=h)
    ls.add(torch.from_numpy(A).to(DEV), torch.from_numpy(b).to(DEV))
    ls.remove(torch.from_numpy(A[m0:]).to(DEV), torch.from_numpy(b[m0:]).to(DEV))
    assert ls.rows == m0
    x = ls.solve().cpu().numpy()
    floor = E.FLOOR_EPS * E.EPS * np.sqrt(m0 + k)
    res = ls.residual_norm().cpu().numpy()
    for r in range(2):
        s = E.nrm(x_e[:, r])
        got, ref = E.nrm(x[:, r] - x_e[:, r]) / s, E.nrm(x64[:, r] - x_e[:, r]) / s
        assert got <= E.C_REL * max(ref, floor), f"x: {got:.3e} vs fp64 oracle {ref:.3e}; rhs {r}"
        res_e = np.linalg.norm(Ar @ x_e[:, r] - br[:, r])
        assert abs(res[r] - res_e) <= 1e-8 * np.linalg.norm(b[:, r]), (res[r], res_e)


def test_sliding_window(D, h):
    """200 000 x 256 in blocks of 12 500 rows through a 50 000-row window: after every slide x and the residual norm match the
    least-squares solution of the window's rows."""
    n, m, blk, win = 256, 200_000, 12_500, 50_000
    A = F.make("normal", m, n, seed=31)
    b = F.rhs(m, 1, seed=32).reshape(m, 1)
    ls = D.StreamingLeastSquares(n, 1, device=0, handle=h)
    for r0 in range(0, m, blk):
        ls.add(torch.from_numpy(A[r0:r0 + blk]).to(DEV), torch.from_numpy(b[r0:r0 + blk]).to(DEV))
        lo = r0 + blk - win
        if lo > 0:
            ls.remove(np.asfortranarray(A[lo - blk:lo]), np.asfortranarray(b[lo - blk:lo]))
        lo = max(lo, 0)
        assert ls.rows == r0 + blk - lo
        if lo == 0:
            continue
        Aw, bw = A[lo:r0 + blk], b[lo:r0 + blk, 0]
        xr, res = np.linalg.lstsq(Aw, bw, rcond=None)[:2]
        x = ls.solve().cpu().numpy()
        assert E.nrm(x - xr) / E.nrm(xr) <= 1e-12, f"window ending at row {r0 + blk}"
        assert abs(float(ls.residual_norm()[0]) - np.sqrt(res[0])) <= 1e-10 * np.sqrt(res[0])


# ---------------------------------------------------------------------------------------------------------------------
# failure
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,bad", ((64, 20), (300, 170), (300, 0)))
def test_failure(D, h, n, bad):
    """Nine real rows and one that was never added (zero before column `bad`, large from it on): info is exactly bad + 1, vtop
    and V2 are zero and alpha NaN from that column on, the rows above it are the downdate of the real rows, R's rows from it on
    are untouched, and the next call on the handle gives the bits of a fresh handle."""
    k = 9
    st, A = start(D, h, "normal", n, k)
    R0 = npy(st.A)[:n, :n].copy()
    Z = np.asfortranarray(A[n + 5:].copy())
    Z = np.asfortranarray(np.vstack([Z, np.zeros((1, n))]))
    Z[k, bad:] = 100.0 * np.linalg.norm(A, 2)
    t = downdate(D, h, st, Z)
    assert int(t.info.item()) == bad + 1
    a1, vt, V2 = st.α.cpu().numpy(), t.vtop.cpu().numpy(), npy(t.B)
    assert np.isnan(a1[bad:]).all() and not np.isnan(a1[:bad]).any()
    assert (vt[bad:] == 0).all() and (V2[:, bad:] == 0).all()
    R1 = npy(st.A)[:n, :n]
    assert np.array_equal(np.triu(R1, 1)[bad:], np.triu(R0, 1)[bad:])
    Rrem = signed(np.linalg.qr(A[:n + 5], mode="r"))
    top = signed(full(R1, np.nan_to_num(a1)))[:bad]
    if bad:
        assert relerr(top, Rrem[:bad]) <= 1e-12
    # the next call on this handle gives the bits of a fresh handle
    st2, A2 = start(D, h, "normal", 100, 40, seed=3)
    Rs, als = st2.A.clone(), st2.α.clone()
    t2 = downdate(D, h, st2, np.asfortranarray(A2[105:]))
    assert int(t2.info.item()) == 0
    hf = D.Handle(0)
    try:
        t3 = D.downdate_rows_((Rs, als), D.to_colmajor(A2[105:], DEV), handle=hf)
        torch.cuda.synchronize()
        assert sb(torch.triu(st2.A[:100], 1), torch.triu(Rs[:100], 1))
        assert sb(st2.α, als) and sb(t2.B, t3.B) and sb(t2.vtop, t3.vtop)
    finally:
        hf.close()


def test_remove_failure_leaves_the_solver_unchanged(D, h):
    n = 64
    A = F.make("normal", 3000, n, seed=5)
    b = F.rhs(3000, 2, seed=6).reshape(3000, 2)
    ls = D.StreamingLeastSquares(n, 2, device=0, handle=h)
    ls.add(torch.from_numpy(A).to(DEV), torch.from_numpy(b).to(DEV))
    before = [ls.A.clone(), ls.α.clone(), ls.c.clone(), ls._ss.clone()]
    rows = ls.rows
    with pytest.raises(ValueError, match="column"):
        ls.remove(10.0 * A[:50], b[:50])                  # rows that were never added
    after = [ls.A, ls.α, ls.c, ls._ss]
    assert all(sb(x, y) for x, y in zip(before, after)) and ls.rows == rows
    ls.remove(A[:50], b[:50])                             # and a valid removal still works
    assert ls.rows == rows - 50


# ---------------------------------------------------------------------------------------------------------------------
# storage, streams, launches, memory, errors, the cap
# ---------------------------------------------------------------------------------------------------------------------
SENTINEL = -7


def run_raw(D, h, n, k, R, alpha, Z, ldr, ldz, off, stream=None):
    """dhqr_qr_downdate_f64 + dhqr_apply_downdate_f64 on NaN-fenced buffers with leading dimensions ldr / ldz, all operands `off`
    elements in; info sits between two sentinel words."""
    nan = float("nan")
    bR = torch.full((off + ldr * n + 8,), nan, dtype=torch.float64, device=DEV)
    Rv = bR[off:off + ldr * n].view(n, ldr).t()
    Rv[:n].copy_(torch.from_numpy(R))
    bZ = torch.full((off + ldz * n + 8,), nan, dtype=torch.float64, device=DEV)
    Zv = bZ[off:off + ldz * n].view(n, ldz).t()
    Zv[:k].copy_(torch.from_numpy(Z))
    ba = torch.full((n + 2 + off,), nan, dtype=torch.float64, device=DEV)
    ba[off + 1:off + 1 + n] = torch.from_numpy(alpha)
    bv = torch.full((n + 2 + off,), nan, dtype=torch.float64, device=DEV)
    bi = torch.full((3,), SENTINEL, dtype=torch.int64, device=DEV)
    bc = torch.full((off + ldr * 2 + 8,), nan, dtype=torch.float64, device=DEV)
    cv = bc[off:off + ldr * 2].view(2, ldr).t()
    cv[:n].copy_(torch.from_numpy(F.rhs(n, 2, seed=4).reshape(n, 2)))
    be = torch.full((off + ldz * 2 + 8,), nan, dtype=torch.float64, device=DEV)
    ev = be[off:off + ldz * 2].view(2, ldz).t()
    ev[:k].copy_(torch.from_numpy(F.rhs(k, 2, seed=6).reshape(k, 2)))
    s = stream or torch.cuda.current_stream()
    lib = D._lib
    lib.call("dhqr_qr_downdate_f64", h.raw, n, k, P(Rv), ldr, P(ba[off + 1:]), P(Zv), ldz, P(bv[off + 1:]), P(bi[1:]), SP(s))
    lib.call("dhqr_apply_downdate_f64", h.raw, n, k, P(Zv), ldz, P(bv[off + 1:]), P(cv), ldr, P(ev), ldz, 2, SP(s))
    torch.cuda.synchronize()
    return bR, bZ, ba, bv, bi, bc, be, (Rv, Zv, cv, ev)


def test_storage_contract(D, h):
    n, k = 161, 290
    st, A = start(D, h, "normal", n, k)
    alpha = st.α.cpu().numpy()
    Rn = np.array(npy(st.A)[:n])
    Rn[np.tril_indices(n, 0)] = np.nan                   # the diagonal and lower part hold reflectors: never read
    Z = np.asfortranarray(A[n + 5:])
    base = None
    for ldr, ldz, off in ((n, k, 0), (n + 7, k + 3, 1), (n + 1, k + 64, 3)):
        bR, bZ, ba, bv, bi, bc, be, (Rv, Zv, cv, ev) = run_raw(D, h, n, k, Rn, alpha, Z, ldr, ldz, off)
        Rh = Rv[:n].cpu().numpy()
        assert np.isnan(Rh[np.tril_indices(n, 0)]).all()
        assert np.isfinite(Rh[np.triu_indices(n, 1)]).all()
        assert bi.tolist() == [SENTINEL, 0, SENTINEL]
        for buf, used in ((bR, [(off + j * ldr, off + j * ldr + n) for j in range(n)]), (bZ, [(off + j * ldz, off + j * ldz + k) for j in range(n)]),
                          (ba, [(off + 1, off + 1 + n)]), (bv, [(off + 1, off + 1 + n)]),
                          (bc, [(off + j * ldr, off + j * ldr + n) for j in range(2)]), (be, [(off + j * ldz, off + j * ldz + k) for j in range(2)])):
            mask = torch.ones(buf.numel(), dtype=torch.bool, device=DEV)
            for a, b in used:
                mask[a:b] = False
            assert torch.isnan(buf[mask]).all(), "a write outside the documented operands"
        res = [torch.triu(Rv[:n], 1).nan_to_num(0.0).contiguous(), Zv[:k].contiguous(), ba[off + 1:off + 1 + n].clone(),
               bv[off + 1:off + 1 + n].clone(), cv[:n].contiguous(), ev[:k].contiguous()]
        if base is None:
            base = res
        else:
            assert all(sb(a, b) for a, b in zip(base, res)), f"bits depend on ldr={ldr} ldz={ldz} offset={off}"


def test_side_stream_gated(D, h, gate):
    """The gated protocol of test_gpu_streams.py on a non-blocking side stream: the calls return with the gate closed, and what
    the stream computes behind it is bitwise the ungated legacy-stream result."""
    n, k = 300, 400
    st, A = start(D, h, "normal", n, k)
    R, al = npy(st.A)[:n, :n], st.α.cpu().numpy()
    Ad = F.make("normal", n + 5 + k, n, seed=9)
    bufs = {"R": (dev(R), dev(R + 0.25)), "alpha": (dev(al), dev(al * 2)), "Z": (dev(A[n + 5:]), dev(Ad[n + 5:])),
            "vtop": (torch.zeros(n, dtype=torch.float64, device=DEV), torch.ones(n, dtype=torch.float64, device=DEV)),
            "info": (torch.zeros(1, dtype=torch.int64, device=DEV), torch.full((1,), 5, dtype=torch.int64, device=DEV)),
            "c": (dev(F.rhs(n, 2, seed=1)), dev(F.rhs(n, 2, seed=2))), "e": (dev(F.rhs(k, 2, seed=3)), dev(F.rhs(k, 2, seed=4)))}

    def fn(w, s):
        D._lib.call("dhqr_qr_downdate_f64", h.raw, n, k, P(w["R"]), n, P(w["alpha"]), P(w["Z"]), k, P(w["vtop"]), P(w["info"]), s)
        D._lib.call("dhqr_apply_downdate_f64", h.raw, n, k, P(w["Z"]), k, P(w["vtop"]), P(w["c"]), n, P(w["e"]), k, 2, s)
    case = Case(fn, bufs, ("R", "alpha", "Z", "vtop", "info", "c", "e"))
    case.reference(h)
    run_gated(case, gate, torch.cuda.Stream(), "downdate + apply on a non-blocking side stream")


@pytest.mark.parametrize("n,k", ((300, 500), (33, 7), (1024, 255)))
def test_launch_accounting(D, h, n, k):
    """The downdate launches what the append launches at the same (n, k), class by class."""
    st, A = start(D, h, "normal", n, k)
    R0, a0 = st.A.clone(), st.α.clone()
    got = {}
    for op in ("append", "downdate"):
        R, al = R0.clone(), a0.clone()
        Z = D.to_colmajor(A[n + 5:], DEV)
        c = torch.zeros(n, dtype=torch.float64, device=DEV)
        e = torch.ones(k, dtype=torch.float64, device=DEV)
        torch.cuda.synchronize()
        with E.options(h, profile=1):
            h.profile_reset()
            l0 = h.launch_count()
            if op == "append":
                D.append_rows_((R, al), Z, handle=h).apply_qt_(c, e)
            else:
                D.downdate_rows_((R, al), Z, handle=h).apply_(c, e)
            torch.cuda.synchronize()
            got[op] = (h.launch_count() - l0, {name: v["count"] for name, v in h.profile().items()})
    assert got["downdate"] == got["append"]


def test_no_memory_left(D):
    def free():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info()[0]
    A = F.make("normal", 4000, 512)
    for cycle in range(3):
        hd = D.Handle(0)
        try:
            ls = D.StreamingLeastSquares(512, 2, device=0, handle=hd)
            ls.add(torch.from_numpy(A).to(DEV), torch.ones((4000, 2), dtype=torch.float64, device=DEV))
            ls.remove(torch.from_numpy(A[:1500]).to(DEV), torch.ones((1500, 2), dtype=torch.float64, device=DEV))
            ls.solve()
            del ls
        finally:
            hd.close()
        if cycle == 0:
            base = free()
    assert abs(free() - base) <= 16 << 20


def test_error_codes(D, h):
    lib = D._lib.load()
    n, k = 64, 40
    R = D.colmajor_empty(n, n, DEV)
    R.zero_()
    a = torch.ones(n + 1, dtype=torch.float64, device=DEV)
    Z = D.colmajor_empty(k, n, DEV)
    Z.zero_()
    v = torch.zeros(n + 1, dtype=torch.float64, device=DEV)
    info = torch.full((2,), SENTINEL, dtype=torch.int64, device=DEV)
    c = torch.zeros(n + 1, dtype=torch.float64, device=DEV)
    e = torch.zeros(k + 1, dtype=torch.float64, device=DEV)
    cap = h.get_option("append_max_rows")
    bad = C.c_void_p(a.data_ptr() + 4)
    s = None
    qa = [h.raw, n, k, P(R), n, P(a), P(Z), k, P(v), P(info), s]
    cases = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, cap + 1)], -4: [(3, None), (3, bad)], -5: [(4, n - 1)],
             -6: [(5, None), (5, bad)], -7: [(6, None), (6, bad), (6, P(R)), (6, P(a))], -8: [(7, k - 1)],
             -9: [(8, None), (8, bad), (8, P(a)), (8, P(Z))],
             -10: [(9, None), (9, C.c_void_p(info.data_ptr() + 4)), (9, P(R)), (9, P(a)), (9, P(Z)), (9, P(v))]}
    for code, subs in cases.items():
        for i, val in subs:
            args = list(qa)
            args[i] = val
            l0 = h.launch_count()
            assert lib.dhqr_qr_downdate_f64(*args) == code, (code, i)
            assert h.launch_count() == l0
    ap = [h.raw, n, k, P(Z), k, P(v), P(c), n, P(e), k, 1, s]
    cases = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, cap + 1)], -4: [(3, None), (3, bad)], -5: [(4, k - 1)],
             -6: [(5, None), (5, bad)], -7: [(6, None), (6, bad), (6, P(Z))], -8: [(7, n - 1)], -9: [(8, None), (8, bad), (8, P(c))],
             -10: [(9, k - 1)], -11: [(10, -1)]}
    for code, subs in cases.items():
        for i, val in subs:
            args = list(ap)
            args[i] = val
            l0 = h.launch_count()
            assert lib.dhqr_apply_downdate_f64(*args) == code, (code, i)
            assert h.launch_count() == l0
    # no-ops write nothing, info included
    l0 = h.launch_count()
    assert lib.dhqr_qr_downdate_f64(h.raw, 0, k, None, 1, None, None, k, None, None, s) == 0
    assert lib.dhqr_qr_downdate_f64(h.raw, n, 0, P(R), n, P(a), None, 1, P(v), P(info), s) == 0
    assert lib.dhqr_apply_downdate_f64(h.raw, n, k, P(Z), k, P(v), P(c), n, P(e), k, 0, s) == 0
    torch.cuda.synchronize()
    assert h.launch_count() == l0 and info.tolist() == [SENTINEL, SENTINEL]


def _multi_rank_job(rank, P_, _marker):
    import dhqr_b200 as D2
    h2 = D2.init_distributed(device=0)
    lib = D2._lib.load()
    x = torch.zeros(64, dtype=torch.float64, device=DEV)
    p = C.c_void_p(x.data_ptr())
    l0 = h2.launch_count()
    codes = [lib.dhqr_qr_downdate_f64(h2.raw, 4, 4, p, 4, p, p, 4, p, p, None),
             lib.dhqr_apply_downdate_f64(h2.raw, 4, 4, p, 4, p, p, 4, p, 4, 1, None)]
    out = {"codes": np.array(codes), "launches": np.array(h2.launch_count() - l0)}
    D2.shutdown_distributed()
    return out


L.JOBS.setdefault("downdate_multi_rank", _multi_rank_job)


def test_multi_rank_handle(tmp_path):
    d, so = L.build()
    try:
        ranks = L.run(2, "downdate_multi_rank", str(tmp_path), so, args=(_multi_rank_job,))
    except L.Skip as e:
        pytest.skip(f"the loopback transport cannot run here: {e}")
    finally:
        shutil.rmtree(d, ignore_errors=True)
    for r, res in enumerate(ranks):
        assert res["codes"].tolist() == [-1, -1] and int(res["launches"]) == 0, f"rank {r}"


def test_at_the_cap(D, h):
    """k = append_max_rows and one row less remove the rows of an appended block exactly; one row more returns -3."""
    n, extra = 64, 300
    cap = h.get_option("append_max_rows")
    A = F.make("normal", cap + extra, n, seed=41)
    for k in (cap, cap - 1):
        R = D.colmajor_empty(n, n, DEV)
        R.zero_()
        al = torch.zeros(n, dtype=torch.float64, device=DEV)
        D.append_rows_((R, al), D.to_colmajor(A[:k], DEV), handle=h)
        D.append_rows_((R, al), D.to_colmajor(A[k:], DEV), handle=h)
        t = D.downdate_rows_((R, al), D.to_colmajor(A[:k], DEV), handle=h)
        torch.cuda.synchronize()
        assert int(t.info.item()) == 0, k
        got = signed(full(npy(R), al.cpu().numpy()))
        ref = signed(np.linalg.qr(A[k:], mode="r"))
        assert relerr(got, ref) <= 1e-10, (k, relerr(got, ref))
    Z = D.colmajor_empty(cap + 1, n, DEV)
    v = torch.zeros(n, dtype=torch.float64, device=DEV)
    info = torch.zeros(1, dtype=torch.int64, device=DEV)
    assert D._lib.load().dhqr_qr_downdate_f64(h.raw, n, cap + 1, P(R), n, P(al), P(Z), cap + 1, P(v), P(info), None) == -3
