"""Solves with the adjoint of a factorisation: dhqr_forwardsolve_{f64,c64} (z = R^{-H} c) and dhqr_solve_adj_{f64,c64} (the
minimum-norm solution y = Q [z; 0] of A^H y = c), and forwardsolve_ / solve_adjoint_ / ldiv_adjoint (run with -m gpu on an H100).

Accuracy follows the extended-precision rule of tests/ext_rule.py on z and on y, each as ||d|| / ||.|| against adj_ext of
tests/adjoint_oracle.py (long double): err_gpu <= 8 max(err_fp64_oracle, 16 eps sqrt(m)), the fp64 oracle being np_forwardsolve / np_solve_adj on the
fp64 oracle's factorisation.  The storage contract (bitwise invariance to ldb, lda and base offset; nothing outside b written),
the stream contract (the gated protocol of test_gpu_streams.py) and the argument errors of include/dhqr.h follow.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import adjoint_oracle as AO
import matrix_families as F
from ext_rule import C_REL, EPS, FLOOR_EPS, SIZE, options
from test_gpu_streams import Case, Gate, P, SP, STREAM_KINDS, dev, run_gated

DEV = "cuda:0"
# triangular: R is a random N(0,1) triangle, whose inverse grows like 2^n, so R^{-T} c of a random c overflows double at
# 2048 x 1024 (the fp64 oracle gives Inf / NaN as well): singular to working precision for the adjoint solve
REAL_FAMILIES = tuple(f for f in F.FAMILIES if f not in F.NAN_FAMILIES and f != "triangular")


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


def _dt(cplx):
    return torch.complex128 if cplx else torch.float64


def factor(D, h, A0, nb=0):
    A = D.to_colmajor(A0, DEV)
    st = D.qr_(A, nb=nb, handle=h)
    return A, st.α


def rhs(m, n, k, cplx, seed=7):
    g = np.random.default_rng([m, n, k, seed])
    c = g.standard_normal((n, k))
    if cplx:
        c = c + 1j * g.standard_normal((n, k))
    return np.asfortranarray(c)


def b_block(D, c, m, ldb, cplx, fill=float("nan")):
    """(m, k) column-major block with leading dimension ldb: rows [0, n) = c, rows [n, m) = fill."""
    n, k = c.shape
    b = D.colmajor_empty(m, k, DEV, lda=ldb, dtype=_dt(cplx))
    b.fill_(fill)
    b[:n] = torch.from_numpy(c).to(DEV)
    return b


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


class Ref:
    """z and y in long double, and the fp64 oracle's z and y, for one input and k right-hand sides."""

    def __init__(self, coracle, oracle, A0, k):
        m, n = A0.shape
        self.cplx = np.iscomplexobj(A0)
        self.A0, self.c = A0, rhs(m, n, k, self.cplx)
        self.z, self.y = AO.adj_ext(A0, self.c)
        if self.cplx:
            h64, a64 = oracle.np_qr_c(A0)
            fs, sa = AO.np_forwardsolve_c, AO.np_solve_adj_c
        else:
            h64, a64 = coracle.qr(A0.copy(order="F"))
            fs, sa = AO.np_forwardsolve, AO.np_solve_adj
        self.z64 = np.stack([fs(h64, a64, self.c[:, j]) for j in range(k)], 1)
        self.y64 = sa(h64, a64, self.c)

    def check(self, z, y, cols, where):
        m = self.A0.shape[0]
        floor = FLOOR_EPS * EPS * SIZE["x"](m)
        for key, got, ext, f64 in (("z", z, self.z, self.z64), ("y", y, self.y, self.y64)):
            e_gpu, e64 = rel(got, ext[:, cols]), rel(f64[:, cols], ext[:, cols])
            assert e_gpu <= C_REL * max(e64, floor), \
                f"{key}: err_gpu {e_gpu:.3e} > {C_REL} x max(err_fp64 {e64:.3e}, floor {floor:.1e}); {where}"


def run_both(D, h, A, alpha, c, m, ldb, cplx, nrhs):
    """forwardsolve_ and solve_adjoint_ on c[:, :nrhs]: (z, y) as numpy, after checking that forwardsolve left rows [n, m) alone."""
    n = c.shape[0]
    cc = c[:, :nrhs]
    if nrhs == 1:
        bf = torch.full((m,), float("nan"), dtype=_dt(cplx), device=DEV)
        bf[:n] = torch.from_numpy(cc[:, 0]).to(DEV)
        by = bf.clone()
    else:
        bf = b_block(D, cc, m, ldb, cplx)
        by = b_block(D, cc, m, ldb, cplx)
    z = D.forwardsolve_(bf, A, alpha, handle=h)
    assert torch.isnan(bf[n:].real).all(), "forwardsolve_ wrote rows n..m-1"
    y = D.solve_adjoint_(by, A, alpha, handle=h)
    assert y is by
    z, y = z.cpu().numpy(), y.cpu().numpy()
    return z.reshape(n, nrhs), y.reshape(m, nrhs)


def residual(A0, y, c):
    """||A^H y - c|| / (||A|| ||y||)."""
    return float(np.linalg.norm(A0.conj().T @ y - c) / (np.linalg.norm(A0) * np.linalg.norm(y)))


_cache = {}


def ref_for(key, make):
    if key not in _cache:
        _cache.clear()
        _cache[key] = make()
    return _cache[key]


# ---------------------------------------------------------------------------------------------------------------------
# 1: accuracy
# ---------------------------------------------------------------------------------------------------------------------
FAMILY_CASES = [(f, w, k) for f in REAL_FAMILIES for w in (1, 0) for k in (1, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("family,wave,nrhs", FAMILY_CASES, ids=[f"{f}-wave{w}-nrhs{k}" for f, w, k in FAMILY_CASES])
def test_adjoint_f64_families(D, h, coracle, oracle, family, wave, nrhs):
    m, n = 2048, 1024
    ref = ref_for(("f64", family), lambda: Ref(coracle, oracle, F.make(family, m, n), 3))
    A, alpha = factor(D, h, ref.A0)
    with options(h, bs_wave=wave):
        z, y = run_both(D, h, A, alpha, ref.c, m, m + 5, False, nrhs)
    ref.check(z, y, slice(0, nrhs), f"Float64 {family} {m}x{n}, bs_wave = {wave}, nrhs = {nrhs}")


@pytest.mark.gpu
@pytest.mark.parametrize("family", F.COMPLEX_FAMILIES)
@pytest.mark.parametrize("nrhs", [1, 3])
def test_adjoint_c64_families(D, h, coracle, oracle, family, nrhs):
    m, n = 1024, 384
    ref = ref_for(("c64", family), lambda: Ref(coracle, oracle, F.make_complex(family, m, n), 3))
    A, alpha = factor(D, h, ref.A0)
    z, y = run_both(D, h, A, alpha, ref.c, m, m + 5, True, nrhs)
    ref.check(z, y, slice(0, nrhs), f"ComplexF64 {family} {m}x{n}, nrhs = {nrhs}")


EDGE_SHAPES = [(300, 1), (300, 31), (300, 32), (300, 33), (300, 127), (300, 129), (200, 200), (201, 200), (1, 1)]
EDGE_CASES = [(m, n, nb) for (m, n) in EDGE_SHAPES for nb in (0, 64, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,nb", EDGE_CASES, ids=[f"{m}x{n}-nb{nb}" for m, n, nb in EDGE_CASES])
def test_adjoint_f64_shape_edges(D, h, coracle, oracle, m, n, nb):
    ref = ref_for(("f64e", m, n), lambda: Ref(coracle, oracle, F.make("normal", m, n), 3))
    A, alpha = factor(D, h, ref.A0, nb)
    for wave in (1, 0):
        with options(h, bs_wave=wave):
            for k in (1, 3):
                z, y = run_both(D, h, A, alpha, ref.c, m, m + 5, False, k)
                where = f"Float64 {m}x{n}, nb = {nb}, bs_wave = {wave}, nrhs = {k}"
                ref.check(z, y, slice(0, k), where)
                assert residual(ref.A0, y, ref.c[:, :k]) < 1e-14, where


@pytest.mark.gpu
@pytest.mark.parametrize("m,n", [(200, 63), (200, 64), (200, 65), (300, 1), (300, 129), (200, 200), (201, 200)])
def test_adjoint_c64_shape_edges(D, h, coracle, oracle, m, n):
    ref = ref_for(("c64e", m, n), lambda: Ref(coracle, oracle, F.make_complex("centered", m, n), 3))
    A, alpha = factor(D, h, ref.A0)
    for k in (1, 3):
        z, y = run_both(D, h, A, alpha, ref.c, m, m + 5, True, k)
        where = f"ComplexF64 {m}x{n}, nrhs = {k}"
        ref.check(z, y, slice(0, k), where)
        assert residual(ref.A0, y, ref.c[:, :k]) < 1e-14, where


# ---------------------------------------------------------------------------------------------------------------------
# 2: properties
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nrhs", [1, 4])
def test_adjoint_f64_range_and_normal_equations(D, h, nrhs):
    m, n = 2048, 1024
    A0 = F.make("normal", m, n)
    A, alpha = factor(D, h, A0)
    c = rhs(m, n, nrhs, False)
    y = D.ldiv_adjoint(D.DistributedHouseholderQRStruct(A, alpha, h), torch.from_numpy(c[:, 0] if nrhs == 1 else c).to(DEV))
    yy = y.reshape(m, nrhs).cpu().numpy()
    assert residual(A0, yy, c) < 1e-14
    # y lies in the range of A: y - Q [(Q'y)[:n]; 0] = 0
    w = y.clone()
    D.apply_qt_(w, A, handle=h)
    w[n:] = 0
    D.apply_q_(w, A, handle=h)
    assert float(torch.linalg.norm(w - y) / torch.linalg.norm(y)) < 1e-14
    # R^{-1} R^{-T} c = (A'A)^{-1} c: forwardsolve_ then backsolve_
    b = torch.zeros(m, dtype=torch.float64, device=DEV)
    b[:n] = torch.from_numpy(c[:, 0]).to(DEV)
    D.forwardsolve_(b, A, alpha, handle=h)
    x = D.backsolve_(b, A, alpha, handle=h).cpu().numpy()
    x_ref = np.linalg.solve(A0.T @ A0, c[:, 0])
    assert rel(x, x_ref) < 1e-10


@pytest.mark.gpu
def test_adjoint_f64_full_size_against_torch(D, h):
    m, n, k = 32768, 4096, 2
    g = torch.Generator(device=DEV).manual_seed(11)
    A0 = D.colmajor_empty(m, n, DEV)
    A0.copy_(torch.rand(m, n, dtype=torch.float64, device=DEV, generator=g))
    c = torch.randn(n, k, dtype=torch.float64, device=DEV, generator=g)
    A = A0.clone()
    H = D.qr_(A, handle=h)
    y = H.ldiv_adjoint(c)
    y1 = H.ldiv_adjoint(c[:, 0])
    a, tau = torch.geqrf(A0)
    z = torch.linalg.solve_triangular(torch.triu(a[:n]).mT, c, upper=False)
    Y = torch.zeros(m, k, dtype=torch.float64, device=DEV)
    Y[:n] = z
    y_t = torch.ormqr(a, tau, Y, left=True, transpose=False)
    for got, want, cc in ((y, y_t, c), (y1, y_t[:, 0], c[:, 0])):
        res = float(torch.linalg.norm(A0.mT @ got - cc) / (torch.linalg.norm(A0) * torch.linalg.norm(got)))
        assert res < 1e-14
        assert float(torch.linalg.norm(got - want) / torch.linalg.norm(want)) < 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# 3: the storage contract
# ---------------------------------------------------------------------------------------------------------------------
def _call(D, name, h, m, n, A, lda, alpha, b, ldb, k, stream=None):
    D._lib.call(name, h.raw, m, n, P(A), lda, P(alpha), P(b), ldb, k, stream)


def _placed(src, ld, off, pad=64):
    """src (m, k) column-major -> (flat NaN-filled buffer, view at element offset off with leading dimension ld)."""
    m, k = src.shape
    buf = torch.full((pad + off + ld * k + pad,), float("nan"), dtype=src.dtype, device=DEV)
    view = buf[pad + off:pad + off + ld * k].view(k, ld).t()[:m]
    view.copy_(src)
    return buf, view


@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", ["forwardsolve", "solve_adj"])
@pytest.mark.parametrize("nrhs", [1, 3])
def test_adjoint_storage_contract(D, h, cplx, name, nrhs):
    m, n = (1000, 300) if cplx else (2048, 1024)
    fn = f"dhqr_{name}_{'c64' if cplx else 'f64'}"
    A0 = F.make_complex("centered", m, n) if cplx else F.make("normal", m, n)
    A, alpha = factor(D, h, A0)
    c = torch.from_numpy(rhs(m, n, nrhs, cplx)).to(DEV)
    b0 = torch.full((m, nrhs), float("nan"), dtype=_dt(cplx), device=DEV)
    b0[:n] = c
    off = 1                                                    # one element: 8 B (Float64) or 16 B (ComplexF64)
    results = []
    for lda in (m, m + 2):
        for aoff in (0, off):
            abuf, Av = _placed(A, lda, aoff)
            albuf, alv = _placed(alpha.reshape(n, 1), n, aoff)
            a_before, al_before = abuf.clone(), albuf.clone()
            for ldb in (m, m + 1, m + 3):
                for boff in (0, off):
                    bbuf, bv = _placed(b0, ldb, boff)
                    before = bbuf.clone()
                    _call(D, fn, h, m, n, Av, lda, alv, bv, ldb, nrhs)
                    torch.cuda.synchronize()
                    where = f"{fn} nrhs = {nrhs}, lda = {lda} + {aoff}, ldb = {ldb} + {boff}"
                    assert torch.equal(abuf.view(torch.uint8), a_before.view(torch.uint8)), f"A changed; {where}"
                    assert torch.equal(albuf.view(torch.uint8), al_before.view(torch.uint8)), f"alpha changed; {where}"
                    # everything outside the m x nrhs operand keeps its bits (NaN sentinels included)
                    mask = torch.ones_like(bbuf, dtype=torch.bool)
                    inner = mask[64 + boff:64 + boff + ldb * nrhs].view(nrhs, ldb)
                    inner[:, :m] = False
                    if name == "forwardsolve":
                        inner[:, n:m] = True                   # rows n..m-1 are neither read nor written
                    assert torch.equal(bbuf[mask].view(torch.uint8), before[mask].view(torch.uint8)), f"wrote outside; {where}"
                    out = bv[:n] if name == "forwardsolve" else bv
                    assert not torch.isnan(out.real).any(), f"a sentinel entered the result; {where}"
                    results.append((where, out.clone()))
    for where, r in results[1:]:
        assert torch.equal(r.reshape(-1).view(torch.uint8), results[0][1].reshape(-1).view(torch.uint8)), \
            f"not bitwise equal to lda = ldb = m, aligned; {where}"


@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True])
def test_adjoint_empty_system_zeroes_b(D, h, cplx):
    m, k = 50, 2
    b = D.colmajor_empty(m, k, DEV, lda=m + 3, dtype=_dt(cplx))
    b.fill_(3.0)
    A = D.colmajor_empty(m, 0, DEV, dtype=_dt(cplx))
    alpha = torch.zeros(0, dtype=_dt(cplx), device=DEV)
    D.solve_adjoint_(b, A, alpha, handle=h)
    assert not b.abs().any()
    b.fill_(3.0)
    D.forwardsolve_(b, A, alpha, handle=h)
    assert (b == 3.0).all()


# ---------------------------------------------------------------------------------------------------------------------
# 4: the stream contract of include/dhqr.h (the gated protocol of test_gpu_streams.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    return Gate()


@pytest.fixture(scope="module")
def streams():
    return {"nonblocking": torch.cuda.Stream(), "high": torch.cuda.Stream(priority=-100), "low": torch.cuda.Stream(priority=100),
            "legacy": torch.cuda.default_stream()}


def adj_case(D, h, name, cplx, nrhs):
    m, n = (1000, 300) if cplx else (2048, 1024)
    A0 = F.make_complex("centered", m, n) if cplx else F.make("normal", m, n)
    A, alpha = factor(D, h, A0)
    torch.cuda.synchronize()
    ldb = m + 1
    cs = [rhs(m, n, nrhs, cplx, seed) for seed in (0, 1)]
    bs = [np.vstack([c, np.zeros((m - n, nrhs), dtype=c.dtype)]) for c in cs]
    bufs = {"A": (dev(A.cpu().numpy()), dev(F.make_complex("centered", m, n, 1) if cplx else F.make("normal", m, n, 1))),
            "alpha": (alpha.clone(), -alpha.clone()),
            "b": (dev(bs[0], ldb), dev(bs[1], ldb))}
    fn_name = f"dhqr_{name}_{'c64' if cplx else 'f64'}"

    def fn(w, st):
        D._lib.call(fn_name, h.raw, m, n, P(w["A"]), m, P(w["alpha"]), P(w["b"]), ldb, nrhs, st)
    return Case(fn, bufs, ("b", "A", "alpha"))


STREAM_CASES = [(name, cplx, k, kind) for name in ("forwardsolve", "solve_adj") for cplx in (False, True) for k in (1, 3)
                for kind in STREAM_KINDS]


@pytest.mark.gpu
@pytest.mark.parametrize("name,cplx,nrhs,kind", STREAM_CASES,
                         ids=[f"{nm}-{'c64' if c else 'f64'}-nrhs{k}-{kd}" for nm, c, k, kd in STREAM_CASES])
def test_adjoint_gated(D, h, gate, streams, name, cplx, nrhs, kind):
    case = adj_case(D, h, name, cplx, nrhs)
    case.reference(h)
    run_gated(case, gate, streams[kind], f"{name} {'c64' if cplx else 'f64'} nrhs = {nrhs} on a {kind} stream")


# ---------------------------------------------------------------------------------------------------------------------
# 5: argument errors
# ---------------------------------------------------------------------------------------------------------------------
class _NullHandle:
    raw = C.c_void_p()


@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", ["forwardsolve", "solve_adj"])
def test_adjoint_errors(D, h, cplx, name):
    dt = _dt(cplx)
    fn = f"dhqr_{name}_{'c64' if cplx else 'f64'}"
    m, n = 40, 30
    A, alpha = factor(D, h, F.make_complex("centered", m, n) if cplx else F.make("normal", m, n))
    b = torch.zeros(m, 2, dtype=dt, device=DEV).t().contiguous().t()
    st = SP(torch.cuda.current_stream())

    def code(*args):
        with pytest.raises(D._lib.DhqrError) as e:
            D._lib.call(fn, *args)
        return e.value.code

    assert code(None, m, n, P(A), m, P(alpha), P(b), m, 2, st) == -1
    assert code(h.raw, -1, 0, P(A), m, P(alpha), P(b), m, 2, st) == -2
    assert code(h.raw, m, -1, P(A), m, P(alpha), P(b), m, 2, st) == -3
    assert code(h.raw, m, m + 1, P(A), m, P(alpha), P(b), m, 2, st) == -3
    assert code(h.raw, m, n, None, m, P(alpha), P(b), m, 2, st) == -4
    assert code(h.raw, m, n, P(A), m - 1, P(alpha), P(b), m, 2, st) == -5
    assert code(h.raw, m, n, P(A), m, None, P(b), m, 2, st) == -6
    assert code(h.raw, m, n, P(A), m, P(alpha), None, m, 2, st) == -7
    assert code(h.raw, m, n, P(A), m, P(alpha), P(b), m - 1, 2, st) == -8
    assert code(h.raw, m, n, P(A), m, P(alpha), P(b), m, -1, st) == -9
    if cplx:
        torch.cuda.synchronize()
        before = h.launch_count()
        b_before = b.clone()
        odd = lambda t: C.c_void_p(t.data_ptr() + 8)
        assert code(h.raw, m, n, odd(A), m, P(alpha), P(b), m, 2, st) == -4
        assert code(h.raw, m, n, P(A), m, odd(alpha), P(b), m, 2, st) == -6
        assert code(h.raw, m, n, P(A), m, P(alpha), odd(b), m, 2, st) == -7
        torch.cuda.synchronize()
        assert h.launch_count() == before, "a rejected call enqueued work"
        assert torch.equal(b, b_before)
    D._lib.call(fn, h.raw, m, n, P(A), m, P(alpha), None, m, 0, st)                     # nrhs = 0: nothing to do
    D._lib.call(fn, h.raw, 0, 0, None, 1, None, P(b), 1, 1, st)                          # m = n = 0
    # the same code through the Python layer, and the Python layer's own checks
    with pytest.raises(D._lib.DhqrError) as e:
        D.solve_adjoint_(b, A, alpha, handle=_NullHandle())
    assert e.value.code == -1
    with pytest.raises(TypeError):
        D.forwardsolve_(torch.zeros(m, dtype=torch.float64 if cplx else torch.complex128, device=DEV), A, alpha, handle=h)
    with pytest.raises(ValueError):
        D.solve_adjoint_(torch.zeros(m - 1, dtype=dt, device=DEV), A, alpha, handle=h)


def test_adjoint_null_handle_without_device():
    import dhqr_b200 as D
    lib = D._lib.load()
    for name in ("dhqr_forwardsolve_f64", "dhqr_forwardsolve_c64", "dhqr_solve_adj_f64", "dhqr_solve_adj_c64"):
        assert getattr(lib, name)(None, 4, 2, None, 4, None, None, 4, 1, None) == -1
    assert b"null handle" in lib.dhqr_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# 6: the Python layer
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True])
def test_ldiv_adjoint_python_layer(D, h, cplx):
    m, n = (1000, 300) if cplx else (2048, 1024)
    A0 = F.make_complex("centered", m, n) if cplx else F.make("normal", m, n)
    A, alpha = factor(D, h, A0)
    H = D.DistributedHouseholderQRStruct(A, alpha, h)
    c = torch.from_numpy(rhs(m, n, 3, cplx)).to(DEV)
    A_b, al_b, c_b = A.clone(), alpha.clone(), c.clone()
    y1, y2 = H.ldiv_adjoint(c), D.ldiv_adjoint(H, c)
    v1 = H.ldiv_adjoint(c[:, 1])
    torch.cuda.synchronize()
    assert torch.equal(A, A_b) and torch.equal(alpha, al_b) and torch.equal(c, c_b)
    assert torch.equal(y1, y2)
    assert y1.shape == (m, 3) and v1.shape == (m,)
    assert torch.equal(v1, y1[:, 1]) or float((v1 - y1[:, 1]).abs().max()) < 1e-13 * float(y1.abs().max())
    assert residual(A0, y1.cpu().numpy(), c.cpu().numpy()) < 1e-14
    with pytest.raises(TypeError):
        D.ldiv_adjoint(D.DistributedHouseholderQRStruct(A.cpu().numpy(), alpha.cpu().numpy(), h), c.cpu().numpy())
    with pytest.raises(ValueError):
        H.ldiv_adjoint(c[:-1])
    with pytest.raises(TypeError):
        H.ldiv_adjoint(c.real if cplx else c.to(torch.complex128))
