"""The explicit thin Q of a factorisation: dhqr_form_q_f64 / dhqr_form_q_c64 and form_q / form_r (run with -m gpu on an H100).

Q = H_1 ... H_n [I_n; 0] is held to the extended-precision rule of tests/ext_rule.py, err_gpu <= 8 max(err_fp64_oracle, 16 eps
sqrt(m)), on two metrics against the long double reference Q_ext:
    Q     max_j ||(Q - Q_ext)[:, j]||        orth  max |Q^H Q - I|  (err_fp64: the same of the fp64 oracle's Q)
The fp64 oracle's Q is the reflector sweep of its own factorisation applied to [I; 0] (q_sweep, conjugating for complex).
Q_ext: Float64 through COracle.qr_ext(want_qb) on the columns e_j (every column up to n = 160, a fixed spread of columns
beyond); ComplexF64 through the complex twin's Q^H applied to I_m (row i of Q is conj(Q^H e_i)[:n]), which costs m
right-hand sides, so the complex rule stops at 1000 x 300 and the larger complex shapes are held to reconstruction,
orthogonality and cuSOLVER's householder_product instead.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import matrix_families as F
from ext_rule import EPS, FLOOR_EPS, C_REL
from test_gpu_streams import Case, Gate, P, SP, STREAM_KINDS, dev, run_gated

DEV = "cuda:0"
SHAPES = [(1000, 300), (2048, 512), (1153, 1025), (1024, 1024), (1000, 1000), (160, 160), (129, 128), (65, 33), (33, 32), (1, 1)]
REAL_FAMILIES = ("uniform", "normal", "graded12", "colscale", "kahan")
CPLX_EXT_SHAPES = [(1000, 300), (160, 160), (129, 128), (65, 64), (130, 129), (65, 33), (33, 32), (1, 1)]
CPLX_BIG_SHAPES = [(2048, 512), (1153, 1025), (1024, 1024), (1000, 1000)]
TOL_REC = 1e-13


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


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def factor(D, h, A0, nb=0):
    """Factor the numpy matrix A0 on the device: (A, alpha), A column-major with lda = m."""
    A = D.to_colmajor(A0, DEV)
    st = D.qr_(A, nb=nb, handle=h)
    return A, st.α


def padded(D, m, n, dtype, extra=1):
    return D.colmajor_empty(m, n, DEV, lda=m + extra, dtype=dtype)


def reconstruction(D, Q, A, alpha, A0):
    """||Q form_r(A, alpha) - A0||_F / ||A0||_F on the device (A: the factored matrix, before an in-place form_q)."""
    R = D.form_r(A, alpha)
    A0d = torch.from_numpy(A0).to(DEV)
    return float(torch.linalg.norm(Q @ R - A0d) / torch.linalg.norm(A0d))


def orth(Q):
    """max |Q^H Q - I| (numpy or torch)."""
    if isinstance(Q, np.ndarray):
        return float(np.abs(Q.conj().T @ Q - np.eye(Q.shape[1])).max())
    return float((Q.mH @ Q - torch.eye(Q.shape[1], dtype=Q.dtype, device=Q.device)).abs().max())


def col_err(Q, Qe, cols):
    return float(np.linalg.norm(Q[:, cols] - Qe, axis=0).max())


def q_sweep(H):
    """H_1 ... H_n [I; 0] in fp64 from the stored reflectors (H_j = I - v_j v_j^H), structured like the library's sweep."""
    m, n = H.shape
    W = np.eye(m, n, dtype=H.dtype)
    for j in range(n - 1, -1, -1):
        v = H[j:, j]
        W[j:, j:] -= np.outer(v, v.conj() @ W[j:, j:])
    return W


def ext_columns(n):
    if n <= 160:
        return np.arange(n)
    return np.unique(np.r_[0:4, 126:130, n - 4:n, np.linspace(0, n - 1, 40).astype(int)])


def to_lapack(V):
    """The library's reflectors v_j (|v_j|^2 = 2, H_j = I - v_j v_j^H) in LAPACK's form: u_j = v_j / v_jj, tau_j = |v_jj|^2."""
    d = torch.diagonal(V)
    U = torch.tril(V, -1) / d + torch.eye(V.shape[0], V.shape[1], dtype=V.dtype, device=V.device)
    return U, (d.abs() ** 2).to(V.dtype)


class RealRef:
    """Q_ext on a column subset (long double) and the fp64 oracle's Q for one real input."""

    def __init__(self, coracle, family, m, n):
        self.A0 = F.make(family, m, n)
        self.cols = ext_columns(n)
        E = np.zeros((m, len(self.cols)), order="F")
        E[self.cols, np.arange(len(self.cols))] = 1.0
        _, _, _, self.Qe, _ = coracle.qr_ext(self.A0, E, want_qb=True)
        H64, _ = coracle.qr(self.A0.copy(order="F"))
        Q64 = q_sweep(H64)
        self.e64 = {"Q": col_err(Q64, self.Qe, self.cols), "orth": orth(Q64)}


class CplxRef:
    """Q_ext (long double, all of it: Q = (Q^H I_m)^H [:, :n]) and the fp64 oracle's Q for one complex input."""

    def __init__(self, coracle, oracle, family, m, n):
        self.A0 = F.make_complex(family, m, n)
        self.cols = np.arange(n)
        _, _, qtb, _ = coracle.qr_ext_c(self.A0, np.eye(m, dtype=np.complex128))
        self.Qe = np.ascontiguousarray(qtb[:n].conj().T)
        H64, _ = oracle.np_qr_c(self.A0)
        Q64 = q_sweep(H64)
        self.e64 = {"Q": col_err(Q64, self.Qe, self.cols), "orth": orth(Q64)}


_cache = {}


def ref_for(key, make):
    """One reference at a time: the parameter lists below keep the cases of one input together."""
    if key not in _cache:
        _cache.clear()
        _cache[key] = make()
    return _cache[key]


def check_rule(ref, Q, m, where):
    floor = FLOOR_EPS * EPS * np.sqrt(m)
    gpu = {"Q": col_err(Q, ref.Qe, ref.cols), "orth": orth(Q)}
    for key in gpu:
        assert gpu[key] <= C_REL * max(ref.e64[key], floor), \
            f"{key}: err_gpu {gpu[key]:.3e} > {C_REL} x max(err_fp64 {ref.e64[key]:.3e}, floor {floor:.1e}); {where}"


def run_both(D, h, A0, nb, dtype):
    """form_q out of place (ldq = m + 1) and in place on the same factorisation; returns (Q_out, Q_in, reconstruction errors)."""
    m, n = A0.shape
    A, alpha = factor(D, h, A0, nb)
    Qo = D.form_q(A, out=padded(D, m, n, dtype), handle=h)
    rec_out = reconstruction(D, Qo, A, alpha, A0)
    R = D.form_r(A, alpha)
    Qi = D.form_q(A, out=A, handle=h)
    assert Qi is A
    A0d = torch.from_numpy(A0).to(DEV)
    rec_in = float(torch.linalg.norm(Qi @ R - A0d) / torch.linalg.norm(A0d))
    return Qo.cpu().numpy(), Qi.cpu().numpy(), rec_out, rec_in


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 2: the extended-precision rule and the reconstruction, every path that stores reflectors
# ---------------------------------------------------------------------------------------------------------------------
REAL_CASES = [(f, m, n, nb) for f in REAL_FAMILIES for (m, n) in SHAPES for nb in (0, 64, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("family,m,n,nb", REAL_CASES, ids=[f"{f}-{m}x{n}-nb{nb}" for f, m, n, nb in REAL_CASES])
def test_form_q_f64_ext_rule(D, h, coracle, family, m, n, nb):
    ref = ref_for((family, m, n, False), lambda: RealRef(coracle, family, m, n))
    Qo, Qi, rec_out, rec_in = run_both(D, h, ref.A0, nb, torch.float64)
    for Q, place, rec in ((Qo, "out of place, ldq = m + 1", rec_out), (Qi, "in place", rec_in)):
        where = f"Float64 {family} {m}x{n}, nb = {nb}, {place}"
        check_rule(ref, Q, m, where)
        assert rec < TOL_REC, f"||QR - A|| / ||A|| = {rec:.3e}; {where}"


CPLX_CASES = [(f, m, n) for f in F.COMPLEX_FAMILIES for (m, n) in CPLX_EXT_SHAPES]


@pytest.mark.gpu
@pytest.mark.parametrize("family,m,n", CPLX_CASES, ids=[f"{f}-{m}x{n}" for f, m, n in CPLX_CASES])
def test_form_q_c64_ext_rule(D, h, coracle, oracle, family, m, n):
    ref = ref_for((family, m, n, True), lambda: CplxRef(coracle, oracle, family, m, n))
    Qo, Qi, rec_out, rec_in = run_both(D, h, ref.A0, 0, torch.complex128)
    for Q, place, rec in ((Qo, "out of place, ldq = m + 1", rec_out), (Qi, "in place", rec_in)):
        where = f"ComplexF64 {family} {m}x{n}, {place}"
        check_rule(ref, Q, m, where)
        assert rec < TOL_REC, f"||QR - A|| / ||A|| = {rec:.3e}; {where}"


BIG_CASES = [(f, m, n) for f in F.COMPLEX_FAMILIES for (m, n) in CPLX_BIG_SHAPES]


@pytest.mark.gpu
@pytest.mark.parametrize("family,m,n", BIG_CASES, ids=[f"{f}-{m}x{n}" for f, m, n in BIG_CASES])
def test_form_q_c64_larger_shapes(D, h, family, m, n):
    """Beyond the complex extended reference's reach: reconstruction, orthogonality at the fp64 oracle's level (n eps), and
    cuSOLVER's ungqr on the same reflectors."""
    A0 = F.make_complex(family, m, n)
    Qo, Qi, rec_out, rec_in = run_both(D, h, A0, 0, torch.complex128)
    A, _ = factor(D, h, A0)
    U, tau = to_lapack(A)
    Qt = torch.linalg.householder_product(U, tau).cpu().numpy()
    for Q, place, rec in ((Qo, "out of place", rec_out), (Qi, "in place", rec_in)):
        where = f"ComplexF64 {family} {m}x{n}, {place}"
        assert rec < TOL_REC, f"||QR - A|| / ||A|| = {rec:.3e}; {where}"
        assert orth(Q) < 1e-12, where
        assert np.abs(Q - Qt).max() < 1e-13, where


# ---------------------------------------------------------------------------------------------------------------------
# 3: bits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cplx,m,n", [(False, 1153, 1025), (False, 2048, 512), (True, 130, 129), (True, 1000, 300)])
def test_form_q_bits(D, h, cplx, m, n):
    A0 = F.make_complex("centered", m, n) if cplx else F.make("normal", m, n)
    dt = torch.complex128 if cplx else torch.float64
    A, _ = factor(D, h, A0)
    A_before = A.clone()
    Q1 = D.form_q(A, handle=h)
    Q2 = D.form_q(A, handle=h)
    D.form_q(A, out=padded(D, m, n, dt), handle=h)
    assert torch.equal(A, A_before), "out of place form_q changed A"
    assert torch.equal(Q1, Q2), "two calls differ"
    # a fresh handle, and a handle whose workspace was sized by a larger Q first
    fresh = D.Handle(0)
    try:
        Qf = D.form_q(A, handle=fresh)
    finally:
        torch.cuda.synchronize()
        fresh.close()
    big = D.Handle(0)
    try:
        B0 = F.make_complex("centered", 2 * m, n + 70) if cplx else F.make("normal", 2 * m, min(n + 300, 2 * m))
        B, _ = factor(D, big, B0)
        D.form_q(B, handle=big)
        Qb = D.form_q(A, handle=big)
    finally:
        torch.cuda.synchronize()
        big.close()
    assert torch.equal(Qf, Q1), "a fresh handle gives other bits"
    assert torch.equal(Qb, Q1), "a handle that formed a larger Q first gives other bits"
    Qi = D.form_q(A, out=A, handle=h)
    assert torch.equal(Qi, Q1), "in place differs from out of place"


# ---------------------------------------------------------------------------------------------------------------------
# 4: cross-checks with Q applied to [I; 0] and with cuSOLVER's householder_product
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("m,n", [(2048, 512), (32768, 4096)])
def test_form_q_f64_cross_checks(D, h, m, n):
    g = torch.Generator(device=DEV).manual_seed(3)
    A0 = D.colmajor_empty(m, n, DEV)
    A0.copy_(torch.rand(m, n, dtype=torch.float64, device=DEV, generator=g))
    A = A0.clone()
    st = D.qr_(A, handle=h)
    Q = D.form_q(A, handle=h)
    E = D.colmajor_empty(m, n, DEV)
    E.copy_(torch.eye(m, n, dtype=torch.float64, device=DEV))
    D.apply_q_(E, A, handle=h)
    U, tau = to_lapack(A)
    Qt = torch.linalg.householder_product(U, tau)
    assert float((Q - E).abs().max()) < 1e-13
    assert float((Q - Qt).abs().max()) < 1e-13
    if m == 32768:
        assert orth(Q) < 1e-12
        R = D.form_r(A, st.α)
        assert float(torch.linalg.norm(Q @ R - A0) / torch.linalg.norm(A0)) < TOL_REC


@pytest.mark.gpu
def test_form_q_c64_full_size(D, h):
    m, n = 4400, 4000
    g = torch.Generator(device=DEV).manual_seed(5)
    A0 = D.colmajor_empty(m, n, DEV, dtype=torch.complex128)
    A0.copy_(torch.complex(torch.rand(m, n, dtype=torch.float64, device=DEV, generator=g),
                           torch.rand(m, n, dtype=torch.float64, device=DEV, generator=g)))
    A = A0.clone()
    st = D.qr_(A, handle=h)
    R = D.form_r(A, st.α)
    Q = D.form_q(A, out=A, handle=h)
    assert orth(Q) < 1e-12
    assert float(torch.linalg.norm(Q @ R - A0) / torch.linalg.norm(A0)) < TOL_REC
    del Q, A, R


# ---------------------------------------------------------------------------------------------------------------------
# 5: the stream contract of include/dhqr.h (the same gated protocol as test_gpu_streams.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    return Gate()


@pytest.fixture(scope="module")
def streams():
    return {"nonblocking": torch.cuda.Stream(), "high": torch.cuda.Stream(priority=-100), "low": torch.cuda.Stream(priority=100),
            "legacy": torch.cuda.default_stream()}


def form_q_case(D, h, cplx, inplace):
    m, n = (1000, 300) if cplx else (2048, 1024)
    make = (lambda s: F.make_complex("centered", m, n, s)) if cplx else (lambda s: F.make("normal", m, n, s))
    facs = []
    for seed in (0, 1):
        A, _ = factor(D, h, make(seed))
        torch.cuda.synchronize()
        facs.append(dev(A.cpu().numpy()))
    name = "dhqr_form_q_c64" if cplx else "dhqr_form_q_f64"
    if inplace:
        bufs = {"A": (facs[0], facs[1])}

        def fn(w, st):
            D._lib.call(name, h.raw, m, n, P(w["A"]), m, P(w["A"]), m, st)
        return Case(fn, bufs, ("A",))
    ldq = m + 1
    bufs = {"A": (facs[0], facs[1]), "Q": (torch.zeros_like(dev(make(0), ldq)), dev(make(1), ldq))}

    def fn(w, st):
        D._lib.call(name, h.raw, m, n, P(w["A"]), m, P(w["Q"]), ldq, st)
    return Case(fn, bufs, ("Q", "A"))


STREAM_CASES = [(cplx, inplace, kind) for cplx in (False, True) for inplace in (False, True) for kind in STREAM_KINDS]


@pytest.mark.gpu
@pytest.mark.parametrize("cplx,inplace,kind", STREAM_CASES,
                         ids=[f"{'c64' if c else 'f64'}-{'inplace' if i else 'outofplace'}-{k}" for c, i, k in STREAM_CASES])
def test_form_q_gated(D, h, gate, streams, cplx, inplace, kind):
    case = form_q_case(D, h, cplx, inplace)
    case.reference(h)
    run_gated(case, gate, streams[kind], f"form_q {'c64' if cplx else 'f64'} {'in place' if inplace else 'out of place'} on a "
                                        f"{kind} stream")


@pytest.mark.gpu
def test_form_q_python_layer_on_current_stream(D, h, gate):
    """form_q under torch.cuda.stream(S) returns with S gated and gives the C-ABI's bits on the legacy stream."""
    m, n = 2048, 1024
    A, _ = factor(D, h, F.make("normal", m, n))
    ref = torch.empty_like(A)
    D._lib.call("dhqr_form_q_f64", h.raw, m, n, P(A), m, P(ref), m, SP(torch.cuda.default_stream()))
    out = torch.empty_like(A)
    D.form_q(A, out=out, handle=h)                     # warm-up
    out.fill_(0.5)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    e = gate.close(s)
    with torch.cuda.stream(s):
        D.form_q(A, out=out, handle=h)
    closed = not e.query()
    torch.cuda.synchronize()
    assert closed, "form_q blocked the host while torch's current stream was gated"
    assert torch.equal(out, ref)


# ---------------------------------------------------------------------------------------------------------------------
# 6: argument errors
# ---------------------------------------------------------------------------------------------------------------------
class _NullHandle:
    raw = C.c_void_p()


@pytest.mark.gpu
@pytest.mark.parametrize("cplx", [False, True])
def test_form_q_errors(D, h, cplx):
    dt = torch.complex128 if cplx else torch.float64
    name = "dhqr_form_q_" + ("c64" if cplx else "f64")
    m, n = 40, 30
    A, _ = factor(D, h, F.make_complex("centered", m, n) if cplx else F.make("normal", m, n))
    Q = D.colmajor_empty(m, n, DEV, dtype=dt)
    big = D.colmajor_empty(m, 2 * n, DEV, dtype=dt)
    esz = 16 if cplx else 8
    st = SP(torch.cuda.current_stream())

    def code(*args):
        with pytest.raises(D._lib.DhqrError) as e:
            D._lib.call(name, *args)
        return e.value.code

    assert code(None, m, n, P(A), m, P(Q), m, st) == -1
    assert code(h.raw, -1, 0, P(A), m, P(Q), m, st) == -2
    assert code(h.raw, m, -1, P(A), m, P(Q), m, st) == -3
    assert code(h.raw, m, m + 1, P(A), m, P(Q), m, st) == -3
    assert code(h.raw, m, n, None, m, P(Q), m, st) == -4
    assert code(h.raw, m, n, P(A), m - 1, P(Q), m, st) == -5
    assert code(h.raw, m, n, P(A), m, None, m, st) == -6
    assert code(h.raw, m, n, P(A), m, P(Q), m - 1, st) == -7
    assert code(h.raw, m, n, P(A), m, C.c_void_p(A.data_ptr() + esz), m, st) == -6       # overlaps A, not A itself
    assert code(h.raw, m, n, P(big), m, P(big), m + 1, st) == -6                         # A itself with another ldq
    D._lib.call(name, h.raw, m, 0, None, m, None, m, st)                                  # n = 0: nothing to do
    # the same codes through form_q
    with pytest.raises(D._lib.DhqrError) as e:
        D.form_q(A, handle=_NullHandle())
    assert e.value.code == -1
    with pytest.raises(D._lib.DhqrError) as e:
        D.form_q(D.colmajor_empty(3, 5, DEV, dtype=dt), handle=h)
    assert e.value.code == -3
    with pytest.raises(D._lib.DhqrError) as e:
        D.form_q(big[:, :n], out=big[:, 1:n + 1], handle=h)                               # shifted by one column
    assert e.value.code == -6
    with pytest.raises(TypeError):
        D.form_q(A.cpu().numpy(), handle=h)
    with pytest.raises(ValueError):
        D.form_q(A, out=D.colmajor_empty(m, n - 1, DEV, dtype=dt), handle=h)
    with pytest.raises(TypeError):
        D.apply_q_(torch.zeros(m, dtype=torch.complex128, device=DEV), D.colmajor_empty(m, n, DEV, dtype=torch.complex128))


def test_form_q_null_handle_without_device():
    import dhqr_b200 as D
    lib = D._lib.load()
    assert lib.dhqr_form_q_f64(None, 4, 2, None, 4, None, 4, None) == -1
    assert lib.dhqr_form_q_c64(None, 4, 2, None, 4, None, 4, None) == -1
    assert b"null handle" in lib.dhqr_last_error()
