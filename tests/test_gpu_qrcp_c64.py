"""ComplexF64 QR with column pivoting (dhqr_qrcp_c64), its basic solution (dhqr_solve_qrcp_c64) and the complete orthogonal
decomposition on it (dhqr_cod_c64, dhqr_solve_cod_c64).

A P = Q R is the unpivoted complex factorisation of A[:, p], so the accuracy yardstick is the extended-precision rule of ext_rule.py
on A[:, p] with the device's permutation (COracle.qr_ext_c).  On top of it: the pivot invariant, LAPACK zgeqp3's permutation on
separated inputs, rank revelation, special inputs, the basic and the minimum-norm solutions against extended references,
composability with the other complex entry points, a matrix taller than any Float64 blocked factorisation, the renorm counter, and
the storage, stream, launch-accounting, memory and argument contracts.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import adjoint_oracle as AO
import cod_c_model as CM
import ext_rule as E
import matrix_families as F
import qrcp_c_model as M
from test_gpu_streams import STREAM_KINDS, Case, Gate, P, SP, dev, run_gated

DEV = "cuda:0"
FAMILIES = tuple(f for f in F.COMPLEX_ALL if f not in F.COMPLEX_NAN_FAMILIES)
SEPARATED = ("colscale", "graded6", "graded12", "rowscale")
TABLE = E.Table("qrcp_c64_ext.md")


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


def qrcp(D, h, A0, lda=None):
    A = D.colmajor_empty(*A0.shape, DEV, lda=lda, dtype=torch.complex128)
    A.copy_(torch.from_numpy(A0))
    st = D.qrcp_(A, handle=h)
    torch.cuda.synchronize()
    return st, npy(A), st.α.cpu().numpy(), st.p.cpu().numpy()


def check_factor(coracle, oracle, path, family, A0, H, alpha, p, k=None):
    Ap = np.asfortranarray(A0[:, p])
    ref = E.Ref(coracle, oracle, family, *Ap.shape, k=k, cplx=True, solve=False, A=Ap)
    gpu, absolute = E.factor_checks(path, ref, H, alpha, f"qrcp_c64 {A0.shape}")
    TABLE.check(path, ref, gpu, ref.e64, absolute)


def check_pivot_invariant(H, alpha):
    R = M.form_r(H, alpha)
    t = np.sqrt(np.cumsum((np.abs(R) ** 2)[::-1], axis=0)[::-1])       # t[k, c] = ||R[k:c+1, c]||
    for k in range(H.shape[1] - 1):
        if abs(alpha[k]) >= 1e-8 * abs(alpha[0]):
            assert abs(alpha[k]) ** 2 >= (1 - 1e-6) * t[k, k + 1:].max() ** 2, f"step {k}: a larger column was left behind"


def crhs(m, k, seed=5):
    return np.asfortranarray(F.rhs(m, k, seed=seed, cplx=True).reshape(m, k))


# ---------------------------------------------------------------------------------------------------------------------
# 1-3: accuracy, the pivot invariant, LAPACK's pivots
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_qrcp_c64_families(D, h, coracle, oracle, family):
    A0 = F.make_complex(family, 2048, 512)
    _, H, alpha, p = qrcp(D, h, A0)
    assert sorted(p) == list(range(512))
    check_factor(coracle, oracle, "qrcp_c64", family, A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n", [(200, 1), (300, 31), (300, 32), (300, 33), (500, 63), (500, 64), (500, 65), (65, 65), (66, 65),
                                 (33, 32), (1, 1)])
def test_qrcp_c64_shape_edges(D, h, coracle, oracle, m, n):
    A0 = F.make_complex("normal", m, n)
    _, H, alpha, p = qrcp(D, h, A0)
    check_factor(coracle, oracle, "qrcp_c64", "normal", A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


@pytest.mark.gpu
def test_qrcp_c64_tall(D, h, coracle, oracle):
    m, n = 728 * h.get_option("sms") + 1000, 64
    A0 = F.make_complex("normal", m, n)
    _, H, alpha, p = qrcp(D, h, A0)
    check_factor(coracle, oracle, "qrcp_c64 tall", "normal", A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


@pytest.mark.gpu
@pytest.mark.parametrize("family", SEPARATED)
def test_qrcp_c64_pivots_match_zgeqp3(D, h, family):
    A0 = F.make_complex(family, 2048, 256)
    _, pl = M.zgeqp3_refformat(A0)
    _, H, alpha, p = qrcp(D, h, A0)
    assert np.array_equal(p, pl)
    Hm, am, pm, _ = M.qrcp_c_model(A0)                                 # and the model's, step for step
    assert np.array_equal(p, pm)


# ---------------------------------------------------------------------------------------------------------------------
# 4-5: rank revelation and special inputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 37, 128, 255])
@pytest.mark.parametrize("noisy", [False, True])
def test_qrcp_c64_rank_revealing(D, h, coracle, oracle, r, noisy):
    m, n = 2048, 256
    A0 = M.low_rank(m, n, r, 1e-13 if noisy else 0.0)
    st, H, alpha, p = qrcp(D, h, A0)
    if noisy:
        assert st.rank(rcond=1e-8) == r
    else:
        assert st.rank() == r
    check_factor(coracle, oracle, f"qrcp_c64 rank {r}{' noisy' if noisy else ''}", "lowrank", A0, H, alpha, p, k=r)


@pytest.mark.gpu
@pytest.mark.parametrize("family", F.COMPLEX_NAN_FAMILIES)
def test_qrcp_c64_zero_column(D, h, family):
    m, n = 2048, 512
    A0 = F.make_complex(family, m, n)
    _, H, alpha, p = qrcp(D, h, A0)
    assert np.isfinite(H).all() and np.isfinite(alpha).all()
    assert p[-1] == F.zero_column(family, n) and alpha[-1] == 0 and not H[n - 1:, n - 1].any()
    assert E.backward_error(np.asfortranarray(A0[:, p[:n - 1]]), H, alpha) < 1e-13


@pytest.mark.gpu
def test_qrcp_c64_zero_matrix_and_nan(D, h):
    _, H, alpha, p = qrcp(D, h, np.zeros((300, 70), dtype=np.complex128, order="F"))
    assert not H.any() and not alpha.any() and np.array_equal(p, np.arange(70))
    A0 = F.make_complex("normal", 300, 70)
    A0[123, 45] = complex(np.nan, 0.0)
    _, H, alpha, p = qrcp(D, h, A0)
    assert np.isnan(alpha[0])


# ---------------------------------------------------------------------------------------------------------------------
# 6: the basic solution
# ---------------------------------------------------------------------------------------------------------------------
def check_basic(D, h, coracle, oracle, A0, r, nrhs, where):
    m, n = A0.shape
    st, H, alpha, p = qrcp(D, h, A0)
    b = crhs(m, nrhs)
    db = D.to_colmajor(b, DEV)
    D.solve_qrcp_(db, st.A, st.α, st.p, r, handle=h)
    x = db.cpu().numpy()[:n]
    assert not x[p[r:]].any(), f"x is not zero off the leading columns; {where}"
    if r == 0:
        return x
    Ak = np.asfortranarray(A0[:, p[:r]])
    _, _, _, x_e = coracle.qr_ext_c(Ak, b)
    H64, a64 = oracle.np_qr_c(Ak)
    floor = E.FLOOR_EPS * E.EPS * E.SIZE["x"](m)
    for k in range(nrhs):
        x64 = oracle.np_ldiv_c(H64, a64, b[:, k].copy())
        scale = E.nrm(x_e[:, k])
        got, e64 = E.nrm(x[p[:r], k] - x_e[:, k]) / scale, E.nrm(x64 - x_e[:, k]) / scale
        assert got <= E.C_REL * max(e64, floor), f"x: {got:.3e} vs fp64 {e64:.3e}; rhs {k}; {where}"
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 31, 32, 33, 200])
def test_solve_qrcp_c64_low_rank(D, h, coracle, oracle, r):
    check_basic(D, h, coracle, oracle, M.low_rank(2048, 256, r), r, 1, f"rank {r}")


@pytest.mark.gpu
@pytest.mark.parametrize("nrhs", [1, 3, 65])
def test_solve_qrcp_c64_full_rank(D, h, coracle, oracle, nrhs):
    A0 = F.make_complex("normal", 1500, 200)
    x = check_basic(D, h, coracle, oracle, A0, 200, nrhs, f"full rank, nrhs {nrhs}")
    st, H, alpha, p = qrcp(D, h, A0)                                   # r = n: dhqr_solve_c64 on A[:, p], permuted back
    b = D.to_colmajor(crhs(1500, nrhs), DEV)
    y = D.solve_householder_(b, st.A, st.α, handle=h).cpu().numpy()
    assert np.abs(x[p] - y).max() <= 1e-12 * np.abs(y).max()


@pytest.mark.gpu
def test_solve_qrcp_c64_rank_zero_and_bad_jpvt(D, h, coracle, oracle):
    m, n = 400, 100
    x = check_basic(D, h, coracle, oracle, F.make_complex("normal", m, n), 0, 2, "rank 0")
    assert not x.any()
    st = D.qrcp_(D.to_colmajor(F.make_complex("normal", m, n), DEV), handle=h)
    pbad = st.p.clone()
    pbad[3], pbad[10] = -1, n                                          # out of range: skipped
    buf = torch.full((m + 64,), complex(float("nan"), float("nan")), dtype=torch.complex128, device=DEV)
    b = buf[32:32 + m]
    b.copy_(torch.from_numpy(F.rhs(m, 1, seed=2, cplx=True)))
    D.solve_qrcp_(b, st.A, st.α, pbad, n, handle=h)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:32]).all() and torch.isnan(buf[32 + m:]).all()


# ---------------------------------------------------------------------------------------------------------------------
# 7: the complete orthogonal decomposition
# ---------------------------------------------------------------------------------------------------------------------
def rr_h(H, alpha, r):
    """R_r^H (n x r) from the computed factorisation: what k_cod_pack_c writes."""
    return np.asfortranarray(M.form_r(H, alpha)[:r].conj().T)


def cod_fp64_c(oracle, A0, p, r, b):
    """The solve's stages in fp64 numpy on the device's permutation and rank: x = P Z [U^{-H} (Q^H b)[0:r]; 0]."""
    m, n = A0.shape
    Ap = np.asfortranarray(A0[:, p])
    H64, a64 = oracle.np_qr_c(Ap)
    G = np.asfortranarray((np.triu(H64[:r], 1) + np.diag(a64)[:r])[:, :n].conj().T)
    HG, aG = oracle.np_qr_c(G)
    x = np.zeros((n, b.shape[1]), dtype=np.complex128)
    for k in range(b.shape[1]):
        c = oracle.np_apply_qt_c(H64[:, :r], b[:, k].copy())[:r]
        x[p, k] = AO.np_solve_adj_c(HG, aG, c.reshape(r, 1))[:, 0]
    return x


def cod_solve(D, h, st, r, b):
    Fd, gd = D.cod_(st.A, st.α, r, handle=h)
    db = D.to_colmajor(b, DEV)
    D.solve_cod_(db, st.A, st.p, Fd, gd, r, handle=h)
    torch.cuda.synchronize()
    return db.cpu().numpy(), Fd, gd


def check_x(oracle, A0, p, r, b, x, where):
    m, n = A0.shape
    x_ext = CM.cod_ext_c(A0, p, r, b)
    x64 = cod_fp64_c(oracle, A0, p, r, b)
    floor = E.FLOOR_EPS * E.EPS * E.SIZE["x"](m)
    for k in range(b.shape[1]):
        scale = E.nrm(x_ext[:, k])
        got, e64 = E.nrm(x[:n, k] - x_ext[:, k]) / scale, E.nrm(x64[:, k] - x_ext[:, k]) / scale
        assert got <= E.C_REL * max(e64, floor), f"x: {got:.3e} vs fp64 twin {e64:.3e}; rhs {k}; {where}"


@pytest.mark.gpu
@pytest.mark.parametrize("family", ("normal", "graded6", "colscale", "kahan", "imag"))
def test_cod_c64_factor(D, h, coracle, oracle, family):
    A0 = F.make_complex(family, 2048, 512)
    st, H, alpha, p = qrcp(D, h, A0)
    r = st.rank()
    assert r > 0
    Fd, gd = D.cod_(st.A, st.α, r, handle=h)
    torch.cuda.synchronize()
    assert tuple(Fd.shape) == (512, r) and tuple(gd.shape) == (r,) and Fd.dtype == torch.complex128
    G = rr_h(H, alpha, r)
    ref = E.Ref(coracle, oracle, family, 512, r, cplx=True, solve=False, A=G)
    gpu, absolute = E.factor_checks("cod_c64", ref, npy(Fd), gd.cpu().numpy(), f"R_r^H of qrcp_c64 {A0.shape}, rank {r}")
    TABLE.check("cod_c64", ref, gpu, ref.e64, absolute)


@pytest.mark.gpu
@pytest.mark.parametrize("r", [1, 31, 32, 33, 37, 63, 64, 65, 128, 129, 255, 256])
@pytest.mark.parametrize("noisy", [False, True])
def test_solve_cod_c64_low_rank(D, h, oracle, r, noisy):
    m, n = 2048, 256
    A0 = M.low_rank(m, n, r, 1e-13 if noisy else 0.0)
    st, H, alpha, p = qrcp(D, h, A0)
    rd = st.rank(rcond=1e-8)
    assert rd == r
    b = crhs(m, 1)
    x, _, _ = cod_solve(D, h, st, rd, b)
    check_x(oracle, A0, p, rd, b, x, f"rank {r}{' noisy' if noisy else ''}")


@pytest.mark.gpu
@pytest.mark.parametrize("r", [37, 128, 200])
def test_solve_cod_c64_minimum_norm(D, h, r):
    m, n = 2048, 256
    A0 = M.low_rank(m, n, r)
    b = F.rhs(m, 1, seed=7, cplx=True)
    st = D.qrcp_(D.to_colmajor(A0, DEV), handle=h)
    assert st.rank() == r
    cs = st.cod()
    assert cs.rank == r and cs.F.dtype == torch.complex128 and cs.γ.dtype == torch.complex128
    A_before = st.A.clone()
    x = cs.ldiv(torch.from_numpy(b).to(DEV)).cpu().numpy()
    assert torch.equal(st.A, A_before)
    x_pinv = CM.pinv_solve_c(A0, b, r)
    assert np.linalg.norm(x - x_pinv) <= 1e-8 * np.linalg.norm(x_pinv)
    Nul = np.linalg.svd(A0)[2][r:].conj().T                           # null-space basis of the exactly rank-r A
    assert np.linalg.norm(Nul.conj().T @ x) <= 1e-10 * np.linalg.norm(x)
    xb, rb = st.ldiv(torch.from_numpy(b).to(DEV))                     # the basic solution
    xb = xb.cpu().numpy()
    assert rb == r and xb.dtype == np.complex128
    res, resb = np.linalg.norm(A0 @ x - b), np.linalg.norm(A0 @ xb - b)
    assert abs(res - resb) <= 1e-10 * np.linalg.norm(b)
    assert np.linalg.norm(x) <= np.linalg.norm(xb)
    xr = cs.ldiv(torch.from_numpy(b.real.copy()).to(DEV)).cpu().numpy()   # a real b is promoted
    assert np.linalg.norm(xr - CM.pinv_solve_c(A0, b.real.astype(np.complex128), r)) <= 1e-8 * np.linalg.norm(xr)


@pytest.mark.gpu
def test_solve_cod_c64_full_rank_matches_basic(D, h, oracle):
    m, n = 1500, 200
    A0 = F.make_complex("normal", m, n)
    st, H, alpha, p = qrcp(D, h, A0)
    b = crhs(m, 2)
    x, _, _ = cod_solve(D, h, st, n, b)
    check_x(oracle, A0, p, n, b, x, "rank n")
    db = D.to_colmajor(b, DEV)
    xq = D.solve_qrcp_(db, st.A, st.α, st.p, n, handle=h).cpu().numpy()
    assert np.abs(x[:n] - xq).max() <= 1e-12 * np.abs(xq).max()


# ---------------------------------------------------------------------------------------------------------------------
# 8: composability with the other complex entry points
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_qrcp_c64_composes(D, h):
    m, n = 1200, 300
    A0 = F.make_complex("graded6", m, n)
    st = D.qrcp_(D.to_colmajor(A0, DEV), handle=h)
    Ap = torch.from_numpy(np.ascontiguousarray(A0)).to(DEV)[:, st.p]
    R = D.form_r(st.A, st.α)
    Q = D.form_q(st.A, handle=h)
    assert float(((Q @ R - Ap).norm(dim=0) / Ap.norm(dim=0)).max()) < 1e-13
    b = torch.from_numpy(F.rhs(m, 1, seed=1, cplx=True)).to(DEV)
    qtb = D.apply_qt_(b.clone(), st.A, handle=h)
    assert float((qtb[:n] - Q.mH @ b).norm() / b.norm()) < 1e-13
    c = torch.zeros(m, dtype=torch.complex128, device=DEV)
    c[:n] = torch.from_numpy(F.rhs(n, 1, seed=4, cplx=True)).to(DEV)
    z = D.forwardsolve_(c.clone(), st.A, st.α, handle=h)
    zr = torch.linalg.solve_triangular(R.mH, c[:n].reshape(-1, 1), upper=False)[:, 0]
    assert float((z - zr).norm() / zr.norm()) < 1e-9
    y = D.solve_adjoint_(c.clone(), st.A, st.α, handle=h)            # the minimum-norm solution of A[:, p]^H y = c
    assert float((Ap.mH @ y - c[:n]).norm() / c[:n].norm()) < 1e-9
    r = 250
    Fd, gd = D.cod_(st.A, st.α, r, handle=h)
    Z = D.form_q(Fd, handle=h)                                        # form_q(F) = Z[:, :r]
    U = D.form_r(Fd, gd)
    Rr = R[:r]
    assert float(((Z @ U - Rr.mH).norm(dim=0) / Rr.mH.norm(dim=0)).max()) < 1e-13
    assert float((Z.mH @ Z - torch.eye(r, dtype=Z.dtype, device=DEV)).abs().max()) < 1e-13


# ---------------------------------------------------------------------------------------------------------------------
# 9: renorms and contracts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_qrcp_c64_renorms(D, h, coracle, oracle):
    A0 = M.nearly_parallel(2048, 256)
    torch.cuda.synchronize()
    r0 = h.get_option("qrcp_renorms")
    _, H, alpha, p = qrcp(D, h, A0)
    assert h.get_option("qrcp_renorms") - r0 >= 1
    check_factor(coracle, oracle, "qrcp_c64", "nearly_parallel", A0, H, alpha, p)
    check_pivot_invariant(H, alpha)


def _placed(src, ld, off, pad=64):
    """src (m x k) in a NaN-filled complex128 buffer at leading dimension ld, starting `off` whole elements (16 B each) further
    on, so every placement stays 16 B aligned."""
    m, k = src.shape
    buf = torch.full((pad + off + ld * k + pad,), complex(float("nan"), float("nan")), dtype=src.dtype, device=DEV)
    view = buf[pad + off:pad + off + ld * k].view(k, ld).t()[:m]
    view.copy_(src)
    return buf, view


def _outside(buf, off, ld, m, k, pad=64):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[pad + off:pad + off + ld * k].view(k, ld)[:, :m] = False
    return mask


@pytest.mark.gpu
def test_qrcp_c64_storage_contract(D, h):
    m, n, nrhs, r = 1100, 150, 3, 140
    A0 = torch.from_numpy(F.make_complex("graded6", m, n)).to(DEV)
    b0 = torch.from_numpy(crhs(m, nrhs, seed=9)).to(DEV)
    st = SP(torch.cuda.current_stream())
    results = []
    for lda in (m, m + 1, m + 2):
        for off in (0, 1):                                             # base one complex element (16 B) further on
            abuf, Av = _placed(A0, lda, off)
            albuf, alv = _placed(torch.zeros(n, 1, dtype=torch.complex128, device=DEV), n, off)
            pbuf = torch.full((64 + off + n + 64,), -7, dtype=torch.int64, device=DEV)
            pv = pbuf[64 + off:64 + off + n]
            fbuf, Fv = _placed(torch.zeros(n, r, dtype=torch.complex128, device=DEV), n + lda - m, off)
            gbuf, gv = _placed(torch.zeros(r, 1, dtype=torch.complex128, device=DEV), r, off)
            a_before, al_before, p_before = abuf.clone(), albuf.clone(), pbuf.clone()
            D._lib.call("dhqr_qrcp_c64", h.raw, m, n, P(Av), lda, P(alv), P(pv), st)
            D._lib.call("dhqr_cod_c64", h.raw, m, n, r, P(Av), lda, P(alv), P(Fv), n + lda - m, P(gv), st)
            bbuf, bv = _placed(b0, m + 1 + off, off)
            b_before = bbuf.clone()
            D._lib.call("dhqr_solve_qrcp_c64", h.raw, m, n, r, P(Av), lda, P(alv), P(pv), P(bv), m + 1 + off, nrhs, st)
            xb = bv.clone()
            bv.copy_(b0)
            D._lib.call("dhqr_solve_cod_c64", h.raw, m, n, r, P(Av), lda, P(pv), P(Fv), n + lda - m, P(gv), P(bv), m + 1 + off,
                        nrhs, st)
            torch.cuda.synchronize()
            where = f"lda {lda}, offset {off}"
            for buf, before, ld, rows, k in ((abuf, a_before, lda, m, n), (albuf, al_before, n, n, 1), (bbuf, b_before, m + 1 + off, m, nrhs)):
                mask = _outside(buf, off, ld, rows, k)
                assert torch.equal(buf[mask].view(torch.uint8), before[mask].view(torch.uint8)), f"wrote outside; {where}"
            for buf, ld, rows, k in ((fbuf, n + lda - m, n, r), (gbuf, r, r, 1)):
                assert torch.isnan(buf[_outside(buf, off, ld, rows, k)]).all(), f"wrote outside F or gamma; {where}"
            pm = torch.ones_like(pbuf, dtype=torch.bool)
            pm[64 + off:64 + off + n] = False
            assert torch.equal(pbuf[pm], p_before[pm]), f"wrote outside jpvt; {where}"
            results.append((where, Av.clone(), alv.clone(), pv.clone(), Fv.clone(), gv.clone(), xb, bv.clone()))
    for where, *rs in results[1:]:
        for a, b in zip(rs, results[0][1:]):
            assert np.ascontiguousarray(a.cpu().numpy()).tobytes() == np.ascontiguousarray(b.cpu().numpy()).tobytes(), \
                f"not bitwise equal; {where}"


@pytest.mark.gpu
def test_qrcp_c64_repeatable(D, h):
    A0 = F.make_complex("colscale", 3000, 400)
    outs = []
    for _ in range(2):
        st, H, alpha, p = qrcp(D, h, A0)
        Fd, gd = D.cod_(st.A, st.α, 300, handle=h)
        b = D.to_colmajor(crhs(3000, 2), DEV)
        D.solve_cod_(b, st.A, st.p, Fd, gd, 300, handle=h)
        b2 = D.to_colmajor(crhs(3000, 2), DEV)
        D.solve_qrcp_(b2, st.A, st.α, st.p, 300, handle=h)
        outs.append((H, alpha, p, npy(Fd), gd.cpu().numpy(), b.cpu().numpy(), b2.cpu().numpy()))
    assert E.digest(*outs[0]) == E.digest(*outs[1])


@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    return Gate()


@pytest.fixture(scope="module")
def streams():
    return {"nonblocking": torch.cuda.Stream(), "high": torch.cuda.Stream(priority=-100), "low": torch.cuda.Stream(priority=100),
            "legacy": torch.cuda.default_stream()}


def qrcp_c64_case(D, h, name):
    m, n, nrhs, r = 700, 96, 2, 90
    cm = lambda s: F.make_complex("normal", m, n, s)
    if name == "qrcp":
        bufs = {"A": (dev(cm(0)), dev(cm(1))),
                "alpha": (torch.zeros(n, dtype=torch.complex128, device=DEV), torch.full((n,), -1.0 + 0j, dtype=torch.complex128, device=DEV)),
                "p": (torch.zeros(n, dtype=torch.int64, device=DEV), torch.full((n,), 5, dtype=torch.int64, device=DEV))}

        def fn(w, st):
            D._lib.call("dhqr_qrcp_c64", h.raw, m, n, P(w["A"]), m, P(w["alpha"]), P(w["p"]), st)
        return Case(fn, bufs, ("A", "alpha", "p"))
    sts = [D.qrcp_(D.to_colmajor(cm(s), DEV), handle=h) for s in (0, 1)]
    cods = [D.cod_(s.A, s.α, r, handle=h) for s in sts]
    torch.cuda.synchronize()
    flat = lambda t: t.t().contiguous().reshape(-1)
    bufs = {"A": tuple(flat(s.A) for s in sts), "alpha": tuple(s.α.clone() for s in sts), "p": tuple(s.p.clone() for s in sts),
            "F": tuple(flat(c[0]) for c in cods), "gamma": tuple(c[1].clone() for c in cods),
            "b": (dev(crhs(m, nrhs, seed=0)), dev(crhs(m, nrhs, seed=1)))}
    if name == "cod":
        def fn(w, st):
            D._lib.call("dhqr_cod_c64", h.raw, m, n, r, P(w["A"]), m, P(w["alpha"]), P(w["F"]), n, P(w["gamma"]), st)
        return Case(fn, bufs, ("F", "gamma", "A", "alpha"))
    if name == "solve_qrcp":
        def fn(w, st):
            D._lib.call("dhqr_solve_qrcp_c64", h.raw, m, n, r, P(w["A"]), m, P(w["alpha"]), P(w["p"]), P(w["b"]), m, nrhs, st)
        return Case(fn, bufs, ("b", "A", "alpha", "p"))

    def fn(w, st):
        D._lib.call("dhqr_solve_cod_c64", h.raw, m, n, r, P(w["A"]), m, P(w["p"]), P(w["F"]), n, P(w["gamma"]), P(w["b"]), m, nrhs, st)
    return Case(fn, bufs, ("b", "A", "F", "gamma", "p"))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAM_KINDS)
@pytest.mark.parametrize("name", ["qrcp", "solve_qrcp", "cod", "solve_cod"])
def test_qrcp_c64_gated(D, h, gate, streams, name, kind):
    case = qrcp_c64_case(D, h, name)
    case.reference(h)
    assert not case.sync_ok, "the complex pivoted calls never synchronise"
    run_gated(case, gate, streams[kind], f"{name}_c64 on a {kind} stream")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["qrcp", "solve_qrcp", "cod", "solve_cod"])
def test_qrcp_c64_profile_counts_every_launch(D, name):
    hd = D.Handle(0)
    try:
        hd.set_option("profile", 1)
        m, n, r, nrhs = 1024, 300, 260, 2
        A0 = D.to_colmajor(M.low_rank(m, n, r, 1e-13), DEV)
        st = D.qrcp_(A0.clone(), handle=hd)
        Fd, gd = D.cod_(st.A, st.α, r, handle=hd)
        b = D.to_colmajor(crhs(m, nrhs), DEV)
        torch.cuda.synchronize()
        hd.profile_reset()
        n0 = hd.launch_count()
        if name == "qrcp":
            D.qrcp_(A0.clone(), handle=hd)
        elif name == "cod":
            D.cod_(st.A, st.α, r, handle=hd)
        elif name == "solve_qrcp":
            D.solve_qrcp_(b, st.A, st.α, st.p, r, handle=hd)
        else:
            D.solve_cod_(b, st.A, st.p, Fd, gd, r, handle=hd)
        torch.cuda.synchronize()
        launched = hd.launch_count() - n0
        prof = hd.profile()
        assert launched > 0
        assert all(prof), f"a profile class without a name: {sorted(prof)}"
        counts = {k: v["count"] for k, v in prof.items() if v["count"]}
        assert sum(counts.values()) == launched, f"{launched} launches, profile counts {counts}"
        if name == "qrcp":
            assert counts.get("k_qrcp_gemv_c") == n and counts.get("k_qrcp_pivot_c") == n, counts
        if name == "cod":
            assert counts.get("k_cod_pack_c") == 1, counts
    finally:
        hd.close()


@pytest.mark.gpu
def test_qrcp_c64_handle_returns_its_device_memory(D):
    m, n, r, nrhs = 8192, 512, 500, 3
    A0 = torch.from_numpy(F.make_complex("normal", m, n)).to(DEV)
    b0 = torch.from_numpy(crhs(m, nrhs)).to(DEV)
    A, b = D.colmajor_empty(m, n, DEV, dtype=torch.complex128), D.colmajor_empty(m, nrhs, DEV, dtype=torch.complex128)
    al = torch.zeros(n, dtype=torch.complex128, device=DEV)
    jp = torch.zeros(n, dtype=torch.int64, device=DEV)
    Fm = D.colmajor_empty(n, r, DEV, dtype=torch.complex128)
    g = torch.zeros(r, dtype=torch.complex128, device=DEV)

    def run(hd):
        call = D._lib.call
        A.copy_(A0)
        call("dhqr_qrcp_c64", hd.raw, m, n, P(A), m, P(al), P(jp), None)
        call("dhqr_cod_c64", hd.raw, m, n, r, P(A), m, P(al), P(Fm), n, P(g), None)
        for k in (1, nrhs):
            b.copy_(b0)
            call("dhqr_solve_cod_c64", hd.raw, m, n, r, P(A), m, P(jp), P(Fm), n, P(g), P(b), m, k, None)
            b.copy_(b0)
            call("dhqr_solve_qrcp_c64", hd.raw, m, n, r, P(A), m, P(al), P(jp), P(b), m, k, None)
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
def test_qrcp_c64_errors(D, h):
    m, n, r = 40, 30, 20
    cz = lambda *s: torch.zeros(*s, dtype=torch.complex128, device=DEV)
    A = D.to_colmajor(F.make_complex("normal", m, n), DEV)
    alpha, p, g = cz(n + 1), torch.zeros(n + 1, dtype=torch.int64, device=DEV), cz(r + 1)
    b = D.colmajor_empty(m + 1, 2, DEV, dtype=torch.complex128)
    b.zero_()
    Fm = D.colmajor_empty(n, r, DEV, dtype=torch.complex128)
    Fm.zero_()
    st = SP(torch.cuda.current_stream())
    odd = lambda t: C.c_void_p(t.data_ptr() + 8)                      # 8 B aligned, not 16
    odd4 = lambda t: C.c_void_p(t.data_ptr() + 4)

    def code(fn, *args):
        with pytest.raises(D._lib.DhqrError) as e:
            D._lib.call(fn, *args)
        return e.value.code

    def bad(fn, args, i, v):
        a = list(args)
        a[i] = v
        return code(fn, *a)

    torch.cuda.synchronize()
    before = h.launch_count()
    snap = [t.clone() for t in (A, alpha, p, b, Fm, g)]
    q = "dhqr_qrcp_c64"
    qa = [h.raw, m, n, P(A), m, P(alpha), P(p), st]
    assert bad(q, qa, 0, None) == -1
    assert bad(q, qa, 1, -1) == -2
    assert bad(q, qa, 2, -1) == -3 and bad(q, qa, 2, m + 1) == -3
    assert bad(q, qa, 3, None) == -4 and bad(q, qa, 3, odd(A)) == -4
    assert bad(q, qa, 4, m - 1) == -5
    assert bad(q, qa, 5, None) == -6 and bad(q, qa, 5, odd(alpha)) == -6
    assert bad(q, qa, 6, None) == -7 and bad(q, qa, 6, odd4(p)) == -7
    s = "dhqr_solve_qrcp_c64"
    sa = [h.raw, m, n, n, P(A), m, P(alpha), P(p), P(b), m + 1, 2, st]
    assert bad(s, sa, 0, None) == -1
    assert bad(s, sa, 1, -1) == -2
    assert bad(s, sa, 2, m + 1) == -3
    assert bad(s, sa, 3, -1) == -4 and bad(s, sa, 3, n + 1) == -4
    assert bad(s, sa, 4, None) == -5 and bad(s, sa, 4, odd(A)) == -5
    assert bad(s, sa, 5, m - 1) == -6
    assert bad(s, sa, 6, None) == -7 and bad(s, sa, 6, odd(alpha)) == -7
    assert bad(s, sa, 7, None) == -8 and bad(s, sa, 7, odd4(p)) == -8
    assert bad(s, sa, 8, None) == -9 and bad(s, sa, 8, odd(b)) == -9
    assert bad(s, sa, 9, m - 1) == -10
    assert bad(s, sa, 10, -1) == -11
    c = "dhqr_cod_c64"
    ca = [h.raw, m, n, r, P(A), m, P(alpha), P(Fm), n, P(g), st]
    assert bad(c, ca, 0, None) == -1
    assert bad(c, ca, 1, -1) == -2
    assert bad(c, ca, 2, m + 1) == -3
    assert bad(c, ca, 3, -1) == -4 and bad(c, ca, 3, n + 1) == -4
    assert bad(c, ca, 4, None) == -5 and bad(c, ca, 4, odd(A)) == -5
    assert bad(c, ca, 5, m - 1) == -6
    assert bad(c, ca, 6, None) == -7 and bad(c, ca, 6, odd(alpha)) == -7
    assert bad(c, ca, 7, None) == -8 and bad(c, ca, 7, odd(Fm)) == -8
    assert bad(c, ca, 7, P(A)) == -8 and bad(c, ca, 7, P(alpha)) == -8          # F overlapping A or alpha
    assert bad(c, ca, 8, n - 1) == -9
    assert bad(c, ca, 9, None) == -10 and bad(c, ca, 9, odd(g)) == -10
    assert bad(c, ca, 9, P(A)) == -10 and bad(c, ca, 9, P(Fm)) == -10           # gamma overlapping A or F
    sc = "dhqr_solve_cod_c64"
    sca = [h.raw, m, n, r, P(A), m, P(p), P(Fm), n, P(g), P(b), m + 1, 2, st]
    assert bad(sc, sca, 0, None) == -1
    assert bad(sc, sca, 1, -1) == -2
    assert bad(sc, sca, 2, m + 1) == -3
    assert bad(sc, sca, 3, -1) == -4 and bad(sc, sca, 3, n + 1) == -4
    assert bad(sc, sca, 4, None) == -5 and bad(sc, sca, 4, odd(A)) == -5
    assert bad(sc, sca, 5, m - 1) == -6
    assert bad(sc, sca, 6, None) == -7 and bad(sc, sca, 6, odd4(p)) == -7
    assert bad(sc, sca, 7, None) == -8 and bad(sc, sca, 7, odd(Fm)) == -8
    assert bad(sc, sca, 8, n - 1) == -9
    assert bad(sc, sca, 9, None) == -10 and bad(sc, sca, 9, odd(g)) == -10
    assert bad(sc, sca, 10, None) == -11 and bad(sc, sca, 10, odd(b)) == -11
    assert bad(sc, sca, 11, m - 1) == -12
    assert bad(sc, sca, 12, -1) == -13
    torch.cuda.synchronize()
    assert h.launch_count() == before, "a rejected call enqueued work"
    for t, t0 in zip((A, alpha, p, b, Fm, g), snap):
        assert torch.equal(t, t0)
    D._lib.call(q, h.raw, 0, 0, None, 1, None, None, st)                        # n = 0: nothing to do
    D._lib.call(s, h.raw, m, n, n, P(A), m, P(alpha), P(p), None, m, 0, st)      # nrhs = 0
    D._lib.call(c, h.raw, m, n, 0, P(A), m, P(alpha), None, n, None, st)         # rank = 0
    torch.cuda.synchronize()
    assert h.launch_count() == before, "a no-op enqueued work"
    with pytest.raises(D._lib.DhqrError) as e:
        D.qrcp_(A, handle=_NullHandle())
    assert e.value.code == -1
    with pytest.raises(TypeError):
        D.qrcp_(A.to(torch.complex64))
