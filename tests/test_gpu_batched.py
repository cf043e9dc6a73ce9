"""The batched QR of many small problems and its solves (dhqr_qr_batched_f64, dhqr_apply_qt_batched_f64, dhqr_apply_q_batched_f64,
dhqr_solve_batched_f64; DESIGN §2.12).

Accuracy: every problem of a batch that holds one matrix of every family of matrix_families.FAMILIES is held to the extended-
precision rule of ext_rule.py (V, R, bwd, orth; Q'b, Qb and x where the reference solves), the zero-column families to the fp64
oracle's NaN pattern, at shapes on both sides of every cluster-size switch up to the limit.  Then: bitwise independence of the
batch, the position, the layout, the base offset, the run and the handle's history; sentinels around every operand; the single-
problem entry points on a batched factorisation; torch.geqrf and torch.linalg.lstsq as comparators; the stream, graph-capture
and launch-count contracts; every error code.

A block of right-hand sides is held to the rule per problem and metric by its normwise error, ||dX||_F / ||X||_F (||B||_F for
Q'b and Qb), against the fp64 oracle's.  Column by column, one of 65 right-hand sides of a 3 x 2 graded problem (x sensitive
to kappa^2 ~ 1e4 there) lands where the oracle's rounding happens to be small and the library's not: that is the luck of one
right-hand side, not the accuracy of the factorisation.

The module also registers the four entry points in test_gpu_history.py's catalogue at import (it sorts before that module, so
pytest imports it first): six 1000 x 24 problems cut from the catalogue's matrix, and their solves."""
import ctypes as C
import shutil

import numpy as np
import pytest
import torch

import dist_loopback as L
import ext_rule as E
import matrix_families as F
import test_gpu_history as HIST
from test_gpu_streams import P, SP, Gate, same_bits as _same_bits

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TABLE = E.Table("batched_ext.md")
SLAB = 24576
# (m, n) -> CTAs per problem: the smallest of 1, 2, 4, 8 whose slabs of ceil(m / cs) rows x n fit 24 576 doubles
SHAPES = {(1, 1): 1, (3, 2): 1, (8, 4): 1, (32, 32): 1, (33, 32): 1, (100, 64): 1, (257, 96): 2, (1024, 24): 1, (1025, 24): 2,
          (1024, 48): 2, (1025, 48): 4, (2048, 48): 4, (2049, 48): 8, (443, 443): 8, (196608, 1): 8}
NRHS = (1, 3, 65)


def cluster_size(m, n):
    cs = 1
    while cs < 8 and -(-m // cs) * n > SLAB:
        cs *= 2
    return cs


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


def same_bits(a, b):
    return _same_bits(a.contiguous(), b.contiguous())


def batch_of(D, mats, lda=None, stride=None):
    m, n = mats[0].shape
    A = D.colmajor_empty_batched(len(mats), m, n, DEV, lda=lda, stride=stride)
    for i, a in enumerate(mats):
        A[i].copy_(torch.from_numpy(np.asarray(a)))
    return A


def rhs_batch(D, bs, ldb=None, stride=None):
    m, k = bs[0].shape
    b = D.colmajor_empty_batched(len(bs), m, k, DEV, lda=ldb, stride=stride)
    for i, x in enumerate(bs):
        b[i].copy_(torch.from_numpy(np.asarray(x)))
    return b


# ---------------------------------------------------------------------------------------------------------------------
# the history catalogue: six 1000 x 24 problems, the column blocks of the catalogue's matrix X["A"] read as one batch
# ---------------------------------------------------------------------------------------------------------------------
HB, HN = 6, 24


def _hist_batch(X):
    return HIST.up(np.asfortranarray(X["A"][:, :HB * HN]))


@HIST.case("qr_batched", "dhqr_qr_batched_f64")
def _hist_qr(h, s, X):
    A, al = _hist_batch(X), HIST.zeros(HB * HN)
    HIST.call("dhqr_qr_batched_f64", h.raw, HIST.M, HN, HB, HIST.P(A), HIST.M, HIST.M * HN, HIST.P(al), HN, HIST.SP(s))
    return {"A": A, "alpha": al}


def _hist_factored(X):
    if "bq_H" not in X:                  # the factorisation, once, on a handle of its own
        hd, sd = D_().Handle(0), torch.cuda.Stream()
        try:
            with torch.cuda.stream(sd):
                o = _hist_qr(hd, sd, X)
            sd.synchronize()
            X["bq_H"], X["bq_alpha"] = o["A"].cpu().numpy(), o["alpha"].cpu().numpy()
        finally:
            hd.close()
    return HIST.up(X["bq_H"]), HIST.up(X["bq_alpha"]), HIST.up(np.asfortranarray(np.tile(X["b3"], (1, HB))))


def _hist_apply(name):
    def run(h, s, X):
        A, al, b = _hist_factored(X)
        args = [h.raw, HIST.M, HN, HB, HIST.P(A), HIST.M, HIST.M * HN]
        if name == "dhqr_solve_batched_f64":
            args += [HIST.P(al), HN]
        HIST.call(name, *args, HIST.P(b), HIST.M, HIST.M * 3, 3, HIST.SP(s))
        return {"b": b}
    return run


for _name in ("apply_qt", "apply_q", "solve"):
    HIST.case(f"{_name}_batched_r3", f"dhqr_{_name}_batched_f64")(_hist_apply(f"dhqr_{_name}_batched_f64"))


def D_():
    import dhqr_b200
    return dhqr_b200


# ---------------------------------------------------------------------------------------------------------------------
# 1. the extended-precision rule, per problem
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(SHAPES), ids=[f"{m}x{n}" for m, n in SHAPES])
def test_ext_rule(D, h, coracle, oracle, shape):
    m, n = shape
    assert cluster_size(m, n) == SHAPES[shape]
    fams = [f for f in F.FAMILIES if np.isfinite(F.make(f, m, n)).all()]
    mats = [F.make(f, m, n) for f in fams]
    refs = []
    for f, a in zip(fams, mats):
        with np.errstate(all="ignore"):
            nan64 = np.isnan(coracle.qr(a.copy(order="F"))[0]).any()
        if nan64 and not (f in F.NAN_FAMILIES and F.zero_column(f, n) > 0):
            refs.append(None)                # a zero first column (zerocol at n = 1, zerorows at 1 x 1): only the NaN pattern
        else:
            refs.append(E.Ref(coracle, oracle, f, m, n, nrhs=max(NRHS)))
    A = batch_of(D, mats)
    st = D.qr_batched_(A, handle=h)
    torch.cuda.synchronize()
    H, al = A.cpu().numpy(), st.α.cpu().numpy()
    for i, (f, ref) in enumerate(zip(fams, refs)):
        Hi, ai = np.asfortranarray(H[i]), al[i]
        if ref is None:
            with np.errstate(all="ignore"):
                H64, a64 = coracle.qr(mats[i].copy(order="F"))
            assert np.array_equal(np.isnan(Hi), np.isnan(H64)) and np.array_equal(np.isnan(ai), np.isnan(a64)), f"{f} {m}x{n}"
            continue
        gpu, absolute = E.factor_checks("batched", ref, Hi, ai, f"problem {i}")
        TABLE.check(f"batched {m}x{n}", ref, gpu, ref.e64, absolute)
    solved = [i for i, r in enumerate(refs) if r is not None and r.solve]
    if not solved:
        return
    for k in NRHS:
        bs = [refs[i].b[:, :k] for i in solved]
        sub = batch_of(D, [H[i] for i in solved])
        alpha = st.α[solved].contiguous()
        got = {}
        for key, fn in (("qtb", lambda b: D.apply_qt_batched_(b, sub, h)), ("qb", lambda b: D.apply_q_batched_(b, sub, h)),
                        ("x", lambda b: D.solve_batched_(b, sub, alpha, h))):
            b = rhs_batch(D, bs)
            fn(b)
            got[key] = b.cpu().numpy()
        for j, i in enumerate(solved):
            ref = refs[i]
            res = {"qtb": got["qtb"][j], "qb": got["qb"][j], "x": got["x"][j][:n]}
            gpu, e64 = {}, {}
            for key in res:
                e = getattr(ref, key + "_e")[:, :k]
                scale = E.nrm(ref.x_e[:, :k]) if key == "x" else E.nrm(ref.b[:, :k])
                gpu[key] = E.nrm(res[key] - e) / scale
                e64[key] = E.nrm(getattr(ref, key + "64")[:, :k] - e) / scale
            TABLE.check(f"batched {m}x{n} nrhs {k}", ref, gpu, e64, note=f"block of {k} right-hand sides")


# ---------------------------------------------------------------------------------------------------------------------
# 2. bitwise: batch, position, layout, base offset, run; sentinels
# ---------------------------------------------------------------------------------------------------------------------
def alone(D, h, a, b=None):
    """(H, alpha, x-block) of one matrix factored and solved as a batch of one in the default layout."""
    A = batch_of(D, [a])
    st = D.qr_batched_(A, handle=h)
    out = [A[0].clone(), st.α[0].clone()]
    if b is not None:
        bb = rhs_batch(D, [b])
        D.solve_batched_(bb, A, st.α, h)
        out.append(bb[0].clone())
    return out


@pytest.mark.parametrize("shape", [(8, 4), (100, 64), (1025, 24), (2049, 48), (443, 443)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_bitwise_layout(D, h, shape):
    m, n = shape
    nb, k = 5, 3
    rng = np.random.default_rng([m, n])
    mats = [rng.standard_normal((m, n)) for _ in range(nb)]
    bs = [rng.standard_normal((m, k)) for _ in range(nb)]
    ref = [alone(D, h, a, b) for a, b in zip(mats, bs)]
    lda, ldb = m + 3, m + 5
    sa, sal, sb = lda * n + 7, n + 2, ldb * k + 3
    order = list(range(nb))[::-1]
    for off in (0, 1):                          # 8 B base offset
        baseA = torch.full((off + nb * sa + 5,), float("nan"), dtype=torch.float64, device=DEV)
        A = baseA[off:off + nb * sa].as_strided((nb, m, n), (sa, 1, lda))
        for p, i in enumerate(order):
            A[p].copy_(torch.from_numpy(mats[i]))
        baseal = torch.full((off + nb * sal + 5,), float("nan"), dtype=torch.float64, device=DEV)
        al = baseal[off:off + nb * sal].as_strided((nb, n), (sal, 1))
        baseb = torch.full((off + nb * sb + 5,), float("nan"), dtype=torch.float64, device=DEV)
        b = baseb[off:off + nb * sb].as_strided((nb, m, k), (sb, 1, ldb))
        for p, i in enumerate(order):
            b[p].copy_(torch.from_numpy(bs[i]))
        keepA, keepal, keepb = baseA.clone(), baseal.clone(), baseb.clone()
        lib = D._lib.load()
        assert lib.dhqr_qr_batched_f64(h.raw, m, n, nb, P(A), lda, sa, P(al), sal, SP(torch.cuda.current_stream())) == 0
        assert lib.dhqr_solve_batched_f64(h.raw, m, n, nb, P(A), lda, sa, P(al), sal, P(b), ldb, sb, k,
                                          SP(torch.cuda.current_stream())) == 0
        torch.cuda.synchronize()
        for p, i in enumerate(order):
            assert same_bits(A[p], ref[i][0]) and same_bits(al[p], ref[i][1]) and same_bits(b[p], ref[i][2]), f"problem {i}, offset {off}"
        for base, keep, inside in ((baseA, keepA, A), (baseal, keepal, al), (baseb, keepb, b)):
            mask = torch.ones_like(base, dtype=torch.bool)
            idx = torch.arange(base.numel(), device=DEV)
            mask[idx[off:].as_strided(inside.shape, inside.stride()).flatten()] = False
            assert torch.isnan(base[mask]).all() and same_bits(base[mask], keep[mask]), "a sentinel changed"
    # a second run on the same input, another batch size
    A2 = batch_of(D, mats[:2])
    st2 = D.qr_batched_(A2, handle=h)
    for i in range(2):
        assert same_bits(A2[i], ref[i][0]) and same_bits(st2.α[i], ref[i][1])


def test_large_batch(D, h):
    """65 537 problems of 64 x 64 (A spans more than 2^31 bytes): a seeded sample of positions equals batch = 1 calls."""
    m = n = 64
    nb = 65537
    g = torch.Generator(device=DEV).manual_seed(5)
    A = D.colmajor_empty_batched(nb, m, n, DEV)
    A.copy_(torch.rand(nb, n, m, device=DEV, dtype=torch.float64, generator=g).transpose(1, 2))
    assert A.numel() * 8 > 2 ** 31
    pos = sorted(set(np.random.default_rng(7).integers(0, nb, 24).tolist()) | {0, nb - 1})
    src = {p: A[p].clone() for p in pos}
    st = D.qr_batched_(A, handle=h)
    for p in pos:
        B = D.colmajor_empty_batched(1, m, n, DEV)
        B[0].copy_(src[p])
        s1 = D.qr_batched_(B, handle=h)
        assert same_bits(A[p], B[0]) and same_bits(st.α[p], s1.α[0]), f"position {p}"


# ---------------------------------------------------------------------------------------------------------------------
# 3. composability and comparators
# ---------------------------------------------------------------------------------------------------------------------
def test_single_problem_entry_points(D, h, coracle, oracle):
    m, n = 257, 96
    fams = ("normal", "graded6", "colscale")
    refs = [E.Ref(coracle, oracle, f, m, n, nrhs=1) for f in fams]
    A0 = batch_of(D, [r.A for r in refs])
    A = batch_of(D, [r.A for r in refs])
    st = D.qr_batched_(A, handle=h)
    x = st.ldiv(torch.from_numpy(np.stack([r.b[:, 0] for r in refs])).to(DEV))
    for i, ref in enumerate(refs):
        Q = D.form_q(A[i], handle=h)
        R = D.form_r(A[i], st.α[i])
        err = ((Q @ R - A0[i]).norm(dim=0) / A0[i].norm(dim=0)).max().item()
        assert err < 1e-13, (fams[i], err)
        assert (Q.T @ Q - torch.eye(n, dtype=torch.float64, device=DEV)).abs().max().item() < 1e-13
        y = torch.from_numpy(ref.b[:, 0].copy()).to(DEV)
        D.apply_qt_(y, A[i], handle=h)
        D.backsolve_(y, A[i], st.α[i], handle=h)
        for name, got in (("backsolve", y[:n]), ("fused", x[i])):
            e, e64 = ref.solve_errors("x", got.cpu().numpy(), 0)
            TABLE.check(f"single-problem {name}", ref, {"x": e}, {"x": e64})


def test_torch_comparators(D, h, coracle):
    m, n, nb = 300, 40, 16
    g = torch.Generator(device=DEV).manual_seed(3)
    M = torch.randn(nb, m, n, device=DEV, dtype=torch.float64, generator=g)
    bb = torch.randn(nb, m, device=DEV, dtype=torch.float64, generator=g)
    A = D.colmajor_empty_batched(nb, m, n, DEV)
    A.copy_(M)
    st = D.qr_batched_(A, handle=h)
    a, tau = torch.geqrf(M)
    R1 = torch.triu(A[:, :n], 1) + torch.diag_embed(st.α)
    R2 = torch.triu(a[:, :n])
    sgn = torch.sign(torch.diagonal(R1, dim1=1, dim2=2)) * torch.sign(torch.diagonal(R2, dim1=1, dim2=2))
    cn = M.norm(dim=1)
    assert ((R1 - sgn[..., None] * R2).abs() / cn[:, None, :]).max().item() < 1e-13
    x, res = st.ldiv(bb, return_residual=True)
    xl = torch.linalg.lstsq(M, bb[..., None], driver="gels").solution[..., 0]
    assert ((x - xl).norm(dim=1) / xl.norm(dim=1)).max().item() < 1e-12
    for i in range(nb):
        Mi = np.asfortranarray(M[i].cpu().numpy())
        Hi, ai = coracle.qr(Mi.copy(order="F"))
        xo = coracle.ldiv(Hi, ai, bb[i].cpu().numpy().copy())
        r = np.linalg.norm(Mi @ xo - bb[i].cpu().numpy())
        assert abs(res[i].item() - r) <= 1e-10 * r, (i, res[i].item(), r)


# ---------------------------------------------------------------------------------------------------------------------
# 4. contracts
# ---------------------------------------------------------------------------------------------------------------------
CM, CN, CB, CK = 512, 32, 300, 2


def contract_inputs(D):
    g = torch.Generator(device=DEV).manual_seed(11)
    A = D.colmajor_empty_batched(CB, CM, CN, DEV)
    A.copy_(torch.randn(CB, CN, CM, device=DEV, dtype=torch.float64, generator=g).transpose(1, 2))
    b = D.colmajor_empty_batched(CB, CM, CK, DEV)
    b.copy_(torch.randn(CB, CK, CM, device=DEV, dtype=torch.float64, generator=g).transpose(1, 2))
    return A, b


def calls(lib, hraw, A, al, b, F_, s):
    """The four entry points on (A, alpha, b) on stream s: qr on F_ (a copy of A), then the three applies."""
    return {"qr": lambda: lib.dhqr_qr_batched_f64(hraw, CM, CN, CB, P(F_), CM, CM * CN, P(al), CN, s),
            "apply_qt": lambda: lib.dhqr_apply_qt_batched_f64(hraw, CM, CN, CB, P(A), CM, CM * CN, P(b), CM, CM * CK, CK, s),
            "apply_q": lambda: lib.dhqr_apply_q_batched_f64(hraw, CM, CN, CB, P(A), CM, CM * CN, P(b), CM, CM * CK, CK, s),
            "solve": lambda: lib.dhqr_solve_batched_f64(hraw, CM, CN, CB, P(A), CM, CM * CN, P(al), CN, P(b), CM, CM * CK, CK, s)}


@pytest.fixture(scope="module")
def factored(D, h):
    A, b = contract_inputs(D)
    st = D.qr_batched_(A, handle=h)
    torch.cuda.synchronize()
    return A, st.α, b


def reference_outputs(D, h, A0, F0, al0, b0):
    lib = D._lib.load()
    out = {}
    for name in ("qr", "apply_qt", "apply_q", "solve"):
        F_, al, b = A0.clone(), al0.clone(), b0.clone()
        assert calls(lib, h.raw, F0, al, b, F_, SP(torch.cuda.current_stream()))[name]() == 0
        torch.cuda.synchronize()
        out[name] = (F_, al) if name == "qr" else (b,)
    return out


@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    return Gate()


@pytest.mark.parametrize("name", ["qr", "apply_qt", "apply_q", "solve"])
def test_gated_side_stream(D, h, factored, gate, name):
    """Behind a closed gate on a non-blocking side stream, the call returns with the gate still closed and computes what the
    ungated call computes."""
    A0, _ = contract_inputs(D)
    F0, al0, b0 = factored
    ref = reference_outputs(D, h, A0, F0, al0, b0)[name]
    g = gate
    s = torch.cuda.Stream()
    lib = D._lib.load()
    F_, al, b = torch.zeros_like(A0), torch.zeros_like(al0), torch.zeros_like(b0)
    F_.copy_(A0)
    torch.cuda.synchronize()
    e = g.close(s)
    with torch.cuda.stream(s):
        b.copy_(b0)
        al.copy_(al0)
        F_.copy_(A0)
        rc = calls(lib, h.raw, F0, al, b, F_, SP(s))[name]()
    closed = not e.query()
    assert rc == 0
    assert closed, f"{name} blocked the host until the caller's stream drained"
    torch.cuda.synchronize()
    got = (F_, al) if name == "qr" else (b,)
    assert all(same_bits(x, y) for x, y in zip(got, ref)), name


def test_graph_capture_fresh_handle(D, factored):
    A0, _ = contract_inputs(D)
    F0, al0, b0 = factored
    h2 = D.Handle(0)
    try:
        lib = D._lib.load()
        F_, al, b = A0.clone(), torch.zeros_like(al0), b0.clone()
        bs = b0.clone()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, capture_error_mode="global"):
            s = SP(torch.cuda.current_stream())
            assert lib.dhqr_qr_batched_f64(h2.raw, CM, CN, CB, P(F_), CM, CM * CN, P(al), CN, s) == 0
            assert lib.dhqr_solve_batched_f64(h2.raw, CM, CN, CB, P(F_), CM, CM * CN, P(al), CN, P(bs), CM, CM * CK, CK, s) == 0
        F_.copy_(A0)
        bs.copy_(b0)
        gr.replay()
        torch.cuda.synchronize()
        F1, al1, b1 = A0.clone(), torch.zeros_like(al0), b0.clone()
        s = SP(torch.cuda.current_stream())
        assert lib.dhqr_qr_batched_f64(h2.raw, CM, CN, CB, P(F1), CM, CM * CN, P(al1), CN, s) == 0
        assert lib.dhqr_solve_batched_f64(h2.raw, CM, CN, CB, P(F1), CM, CM * CN, P(al1), CN, P(b1), CM, CM * CK, CK, s) == 0
        torch.cuda.synchronize()
        assert same_bits(F_, F1) and same_bits(al, al1) and same_bits(bs, b1)
        assert same_bits(F1, F0) and same_bits(al1, al0)
    finally:
        torch.cuda.synchronize()
        h2.close()


def test_history_and_launch_count(D, factored):
    A0, _ = contract_inputs(D)
    F0, al0, b0 = factored
    h2 = D.Handle(0)
    try:
        first = reference_outputs(D, h2, A0, F0, al0, b0)
        # other entry points and larger batched calls
        M = D.colmajor_empty(2000, 300, DEV)
        D.fill_uniform_(M, 3, handle=h2)
        st = D.qr_(M, handle=h2)
        D.ldiv(st, torch.ones(2000, dtype=torch.float64, device=DEV))
        big = D.colmajor_empty_batched(2 * CB, 4096, 48, DEV)
        big.normal_()
        D.qr_batched_(big, handle=h2)
        torch.cuda.synchronize()
        lib = D._lib.load()
        again = {}
        for name in ("qr", "apply_qt", "apply_q", "solve"):
            F_, al, b = A0.clone(), al0.clone(), b0.clone()
            l0 = h2.launch_count()
            assert calls(lib, h2.raw, F0, al, b, F_, SP(torch.cuda.current_stream()))[name]() == 0
            assert h2.launch_count() == l0 + 1, name
            torch.cuda.synchronize()
            again[name] = (F_, al) if name == "qr" else (b,)
        for name in first:
            assert all(same_bits(x, y) for x, y in zip(first[name], again[name])), name
        with E.options(h2, profile=1):
            F_, al, b = A0.clone(), al0.clone(), b0.clone()
            for name, fn in calls(lib, h2.raw, F0, al, b, F_, SP(torch.cuda.current_stream())).items():
                assert fn() == 0
            prof = h2.profile()
            for cls in ("k_qr_batched", "k_apply_qt_batched", "k_apply_q_batched", "k_solve_batched"):
                assert prof[cls]["count"] == 1, (cls, prof)
    finally:
        torch.cuda.synchronize()
        h2.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. errors
# ---------------------------------------------------------------------------------------------------------------------
def test_errors(D, h):
    lib = D._lib.load()
    lim = h.get_option("batch_max_elems")
    assert lim == 196608
    m, n, nb, k = 16, 4, 3, 2
    buf = torch.zeros(4 * (nb * m * n + nb * m * k + nb * n) + 64, dtype=torch.float64, device=DEV)
    A, al, b = P(buf), C.c_void_p(buf.data_ptr() + 8 * nb * m * n), C.c_void_p(buf.data_ptr() + 8 * (nb * m * n + nb * n))
    mis = C.c_void_p(buf.data_ptr() + 4)
    s = SP(torch.cuda.current_stream())
    qr = [h.raw, m, n, nb, A, m, m * n, al, n, s]
    ap = [h.raw, m, n, nb, A, m, m * n, b, m, m * k, k, s]
    so = [h.raw, m, n, nb, A, m, m * n, al, n, b, m, m * k, k, s]
    big = lim // 64 + 1
    common = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, m + 1)], -4: [(3, -1), (3, 2 ** 31)], -5: [(4, None), (4, mis)],
              -6: [(5, m - 1)], -7: [(6, m * n - 1)]}
    table = {
        "dhqr_qr_batched_f64": (qr, {**common, -8: [(7, None), (7, mis), (7, A)], -9: [(8, n - 1)]}),
        "dhqr_apply_qt_batched_f64": (ap, {**common, -8: [(7, None), (7, mis), (7, A)], -9: [(8, m - 1)], -10: [(9, m * k - 1)],
                                           -11: [(10, -1)]}),
        "dhqr_apply_q_batched_f64": (ap, {**common, -8: [(7, None), (7, mis), (7, A)], -9: [(8, m - 1)], -10: [(9, m * k - 1)],
                                          -11: [(10, -1)]}),
        "dhqr_solve_batched_f64": (so, {**common, -8: [(7, None), (7, mis), (7, A)], -9: [(8, n - 1)],
                                        -10: [(9, None), (9, mis), (9, A), (9, al)], -11: [(10, m - 1)], -12: [(11, m * k - 1)],
                                        -13: [(12, -1)]}),
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
                assert f(*a) == code, (fn, code, idx, val, D._lib.load().dhqr_last_error())
        # no-ops: batch = 0, n = 0, nrhs = 0
        for idx in (3, 2) + ((len(args) - 2,) if fn != "dhqr_qr_batched_f64" else ()):
            a = list(args)
            a[idx] = 0
            assert f(*a) == 0, (fn, idx)
    assert h.launch_count() == l0
    # the size limit: m x 1 with m = batch_max_elems is accepted (the call runs on a batch of one), one row more is -3, and so is
    # a 64-column problem one row past the limit
    col = torch.zeros(lim + 1, dtype=torch.float64, device=DEV)
    x = torch.zeros(lim + 2, dtype=torch.float64, device=DEV)
    lims = {"dhqr_qr_batched_f64": lambda M, N: [h.raw, M, N, 1, P(col), M, M * N, P(x), N, s],
            "dhqr_apply_qt_batched_f64": lambda M, N: [h.raw, M, N, 1, P(col), M, M * N, P(x), M, M, 1, s],
            "dhqr_apply_q_batched_f64": lambda M, N: [h.raw, M, N, 1, P(col), M, M * N, P(x), M, M, 1, s],
            "dhqr_solve_batched_f64": lambda M, N: [h.raw, M, N, 1, P(col), M, M * N, P(x[:1]), N, P(x[1:]), M, M, 1, s]}
    for fn, mk in lims.items():
        f = getattr(lib, fn)
        l1 = h.launch_count()
        assert f(*mk(lim, 1)) == 0 and h.launch_count() == l1 + 1, fn
        l1 = h.launch_count()
        assert f(*mk(lim + 1, 1)) == -3 and f(*mk(big, 64)) == -3 and h.launch_count() == l1, fn
    torch.cuda.synchronize()
    assert same_bits(buf, keep)
    with pytest.raises(ValueError, match="batch_max_elems"):
        D.qr_batched_(D.colmajor_empty_batched(1, 444, 443, DEV), handle=h)
    with pytest.raises(ValueError):
        D.qr_batched_(torch.zeros(2, 8, 4, dtype=torch.float64, device=DEV), handle=h)   # row-major matrices


def _multi_rank_job(rank, P_, _marker):
    import dhqr_b200 as D2
    h2 = D2.init_distributed(device=0)
    lib = D2._lib.load()
    x = torch.zeros(256, dtype=torch.float64, device=DEV)
    p = C.c_void_p(x.data_ptr())
    q = C.c_void_p(x.data_ptr() + 8 * 128)
    l0 = h2.launch_count()
    codes = [lib.dhqr_qr_batched_f64(h2.raw, 4, 4, 1, p, 4, 16, q, 4, None),
             lib.dhqr_apply_qt_batched_f64(h2.raw, 4, 4, 1, p, 4, 16, q, 4, 4, 1, None),
             lib.dhqr_apply_q_batched_f64(h2.raw, 4, 4, 1, p, 4, 16, q, 4, 4, 1, None),
             lib.dhqr_solve_batched_f64(h2.raw, 4, 4, 1, p, 4, 16, q, 4, C.c_void_p(x.data_ptr() + 8 * 192), 4, 4, 1, None)]
    out = {"codes": np.array(codes), "launches": np.array(h2.launch_count() - l0)}
    D2.shutdown_distributed()
    return out


L.JOBS.setdefault("batched_multi_rank", _multi_rank_job)


def test_multi_rank_handle(tmp_path):
    d, so = L.build()
    try:
        ranks = L.run(2, "batched_multi_rank", str(tmp_path), so, args=(_multi_rank_job,))
    except L.Skip as e:
        pytest.skip(f"the loopback transport cannot run here: {e}")
    finally:
        shutil.rmtree(d, ignore_errors=True)
    for r, res in enumerate(ranks):
        assert res["codes"].tolist() == [-1, -1, -1, -1] and int(res["launches"]) == 0, f"rank {r}"
