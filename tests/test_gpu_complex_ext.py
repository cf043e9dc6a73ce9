"""The ComplexF64 path against the extended-precision rule of tests/ext_rule.py on every complex matrix family (run with -m gpu
on an H100).

The complex path has code of its own: the column-by-column panel (k_house1_c, k_apply1_c), the packing of its reflectors for
the real view (k_pack_c), the trailing update as a real block reflector on the real view (the GEMM pair, k_gemm_cvy_p in CTA
pairs included), the back-substitution (k_backsolve_step_c) and the forward substitution with R^H (k_forwardsolve_step_c).
Each is held here to err_gpu <= 8 max(err_fp64_oracle, FLOOR) against the long double oracle (COracle.qr_ext_c, and
adjoint_oracle.adj_ext for the adjoint solves), on the families of tests/matrix_families.py (F.COMPLEX_ALL) at 1024 x 384 and
777 x 321 (321 = 5 * 64 + 1: the last panel is one column wide), after checking that the two oracles describe the same
factorisation.  Beyond the rule:
    zerolead         every pivot an exact +0: alpha_j real and negative, v_jj = 1 to an ulp, v_j exactly zero on rows j+1..n-1
    zerolead_neg*    A[0, 0] = -0 +- 0i: alpha_0 = s (1, -+sin(pi)) as the numpy oracle has it (angle(-0 +- 0i) = +-pi, S:9)
    tall             728 min(SMs, 160) + 1000 rows, taller than any blocked Float64 factorisation
    large            16384 x 2048: two panels held to the rule, the backward error over all columns
    bitwise          qr, apply_qt (65 right-hand sides), form_q and solve_adj do not depend on cvy_persist or on the run
The worst ratio per path and family goes to build/test_gpu_complex_ext_ratios.md.
"""
import numpy as np
import pytest
import torch

import adjoint_oracle as AO
import matrix_families as F
from ext_rule import C_REL, EPS, FLOOR_EPS, Ref, Table, backward_error, digest, factor_checks, nrm, options, run_qr
from test_gpu_form_q import CplxRef, check_rule, orth, q_sweep

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(1024, 384), (777, 321)]
PATHS = ("qr_c64", "solve_c64", "adjoint_c64", "form_q_c64")
NRHS = 3
# triangular: R^{-H} c of a random N(0,1) triangle overflows (test_gpu_adjoint.py); the zero-column families have no solution
NO_ADJOINT = ("triangular",) + F.COMPLEX_NAN_FAMILIES
TOL_REC = 1e-13

TABLE = Table("test_gpu_complex_ext_ratios.md")
check = TABLE.check


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    TABLE.write()


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="module")
def h(D):
    return D.default_handle(0)


class Entry:
    """Everything one (family, shape) needs, made once: the factorisation references (Ref, with NRHS right-hand sides), the
    adjoint references (adj_ext and the fp64 oracle's z, y) and the fp64 oracle's Q."""

    def __init__(self, coracle, oracle, family, m, n):
        self.ref = Ref(coracle, oracle, family, m, n, cplx=True, nrhs=NRHS, keep_h64=True)
        self.kappa = self.ref.check_oracles_agree()
        self.adj = None
        if family not in NO_ADJOINT:
            g = np.random.default_rng([m, n, 17])
            c = np.asfortranarray(g.standard_normal((n, NRHS)) + 1j * g.standard_normal((n, NRHS)))
            z, y = AO.adj_ext(self.ref.A, c)
            H64, a64 = self.ref.H64, self.ref.a64
            self.adj = (c, z, y, np.stack([AO.np_forwardsolve_c(H64, a64, c[:, r]) for r in range(NRHS)], 1),
                        AO.np_solve_adj_c(H64, a64, c))
        self.orth64 = None
        if family not in F.COMPLEX_NAN_FAMILIES:
            self.orth64 = orth(q_sweep(self.ref.H64))
        del self.ref.H64


_cache = {}


def entry(coracle, oracle, family, m, n):
    """One entry at a time: the cases of one (family, shape) run back to back."""
    key = (family, m, n)
    if key not in _cache:
        _cache.clear()
        _cache[key] = Entry(coracle, oracle, family, m, n)
    return _cache[key]


def factor(D, A0, h):
    dA, st, note, _ = run_qr(D, A0, handle=h)
    return dA, st.α, note


def zerolead_exact(family, H, alpha, n, where):
    """zerolead: every pivot is an exact +0 (matrix_families), so alpha_j = -s_j with a zero imaginary part, v_jj = (0 - alpha_j) / s_j
    = 1 to an ulp, and v_j is exactly zero on rows j+1..n-1.  In the zerolead_neg variants only step 0 differs."""
    j0 = 0 if family == "zerolead" else 1
    a = alpha[j0:]
    bad = np.nonzero(~((a.real < 0) & (a.imag == 0)))[0]
    assert bad.size == 0, f"alpha_{bad[0] + j0} = {a[bad[0]]!r} is not real and negative; {where}"
    d = np.diagonal(H)[j0:]
    assert np.abs(d.real - 1.0).max() <= EPS and not d.imag.any(), f"v_jj is not 1 to an ulp; {where}"
    for j in range(n):
        assert not np.abs(H[j + 1:n, j]).any(), f"v_{j} is not exactly zero on rows {j + 1}..{n - 1}; {where}"


def signed_zero_pivot(ref, alpha, where):
    """alpha_0 of A[0, 0] = -0 +- 0i: s (1, -+sin(pi)) (angle = +-pi), as the numpy oracle has it, to the few ulps by which two
    orders of summing the column's squares differ."""
    want = ref.a64[0]
    im_sign = -1.0 if ref.family == "zerolead_neg" else 1.0
    assert want.real > 0 and np.sign(want.imag) == im_sign and abs(abs(want.imag / want.real) - 1.2246467991473532e-16) < 1e-30
    got = alpha[0]
    for part, g, w in (("real", got.real, want.real), ("imaginary", got.imag, want.imag)):
        assert abs(g - w) <= 4 * np.spacing(abs(w)), f"alpha_0 {part} part {g!r} != numpy oracle's {w!r}; {where}"


# ---------------------------------------------------------------------------------------------------------------------
# every family at both shapes: one reference, four paths
# ---------------------------------------------------------------------------------------------------------------------
CASES = [(m, n, f, p) for (m, n) in SHAPES for f in F.COMPLEX_ALL for p in PATHS]


@pytest.mark.parametrize("m,n,family,path", CASES, ids=[f"{m}x{n}-{f}-{p}" for m, n, f, p in CASES])
def test_family(D, h, coracle, oracle, m, n, family, path):
    e = entry(coracle, oracle, family, m, n)
    ref = e.ref
    dA, alpha, note = factor(D, ref.A, h)
    note += f"; kappa {e.kappa:.2e}"
    where = f"{family} {m}x{n}, {path}"
    if path == "qr_c64":
        H, al = dA.cpu().numpy(), alpha.cpu().numpy()
        gpu, absolute = factor_checks(path, ref, H, al, note)
        check(path, ref, gpu, ref.e64, absolute, note)
        if family in F.ZEROLEAD:
            zerolead_exact(family, H, al, n, where)
        if family in ("zerolead_neg", "zerolead_negneg"):
            signed_zero_pivot(ref, al, where)
    elif path == "solve_c64":
        if not ref.solve:
            pytest.skip("the zero-column families have no solution")
        B = torch.from_numpy(ref.b).to(DEV)
        b0 = B[:, 0].contiguous()
        qtb1 = D.apply_qt_(b0.clone(), dA, handle=h).cpu().numpy()
        x1 = D.ldiv(D.DistributedHouseholderQRStruct(dA, alpha, h), b0).cpu().numpy()
        Q3 = D.colmajor_empty(m, NRHS, DEV, lda=m + 3, dtype=torch.complex128)
        Q3.copy_(B)
        D.apply_qt_(Q3, dA, handle=h)
        X3 = D.colmajor_empty(m, NRHS, DEV, lda=m + 3, dtype=torch.complex128)
        X3.copy_(B)
        X3 = D.solve_householder_(X3, dA, alpha, handle=h).cpu().numpy()
        Q3 = Q3.cpu().numpy()
        for label, qtb, x, r in [("nrhs=1", qtb1, x1, 0)] + [(f"nrhs=3 (rhs {r})", Q3[:, r], X3[:, r], r) for r in range(NRHS)]:
            gpu, e64 = {}, {}
            for key, got in (("qtb", qtb), ("x", x)):
                gpu[key], e64[key] = ref.solve_errors(key, got, r)
            check(f"apply_qt/solve_c64 {label}", ref, gpu, e64, note=note)
    elif path == "adjoint_c64":
        if e.adj is None:
            pytest.skip("no adjoint solution to compare (see NO_ADJOINT)")
        c, z_e, y_e, z64, y64 = e.adj
        for k in (1, NRHS):
            bf = D.colmajor_empty(m, k, DEV, lda=m + 5, dtype=torch.complex128)
            bf.fill_(float("nan"))
            bf[:n] = torch.from_numpy(c[:, :k]).to(DEV)
            by = bf.clone()
            if k == 1:
                bf, by = bf[:, 0].contiguous(), by[:, 0].contiguous()
            z = D.forwardsolve_(bf, dA, alpha, handle=h).cpu().numpy().reshape(n, k)
            assert torch.isnan(bf[n:].real).all(), f"forwardsolve_ wrote rows n..m-1; {where}"
            y = D.solve_adjoint_(by, dA, alpha, handle=h).cpu().numpy().reshape(m, k)
            for r in range(k):
                for key, got, ext, f64 in (("forwardsolve", z, z_e, z64), ("solve_adj", y, y_e, y64)):
                    scale = nrm(ext[:, r])
                    check(f"{key}_c64 nrhs={k}", ref, {"x": nrm(got[:, r] - ext[:, r]) / scale},
                          {"x": nrm(f64[:, r] - ext[:, r]) / scale}, note=note)
    else:
        if e.orth64 is None:
            pytest.skip("a zero column makes Q NaN from that column on")
        Q = D.form_q(dA, handle=h)
        floor = FLOOR_EPS * EPS * np.sqrt(m)
        o = orth(Q)
        assert o <= C_REL * max(e.orth64, floor), \
            f"orth: err_gpu {o:.3e} > {C_REL} x max(err_fp64 {e.orth64:.3e}, floor {floor:.1e}); {where}"
        A0 = torch.from_numpy(ref.A).to(DEV)
        rec = ((Q @ D.form_r(dA, alpha) - A0).norm(dim=0) / A0.norm(dim=0)).max().item()
        assert rec < TOL_REC, f"max_j ||(QR - A)[:, j]|| / ||A[:, j]|| = {rec:.3e}; {where}"


@pytest.mark.parametrize("family", [f for f in F.COMPLEX_ALL if f not in F.COMPLEX_NAN_FAMILIES])
def test_form_q_ext(D, h, coracle, oracle, family):
    # the Q_ext rule of test_gpu_form_q.py (every column of Q against the long double Q, and orthogonality) on every family
    m, n = 300, 128
    ref = CplxRef(coracle, oracle, family, m, n)
    A = D.to_colmajor(ref.A0, DEV)
    D.qr_(A, handle=h)
    Q = D.form_q(A, out=D.colmajor_empty(m, n, DEV, lda=m + 1, dtype=torch.complex128), handle=h).cpu().numpy()
    check_rule(ref, Q, m, f"ComplexF64 {family} {m}x{n}")


# ---------------------------------------------------------------------------------------------------------------------
# past the Float64 row limit, and two full panels at scale
# ---------------------------------------------------------------------------------------------------------------------
def test_tall(D, h, coracle, oracle):
    # the blocked Float64 path stops at 728 min(SMs, 160) rows (test_gpu_ext.py::test_row_limit); the complex path has no limit
    m, n = 728 * min(h.get_option("sms"), 160) + 1000, 128
    ref = Ref(coracle, oracle, "normal", m, n, cplx=True, keep_h64=True)
    ref.check_oracles_agree()
    dA, alpha, note = factor(D, ref.A, h)
    where = f"tall m={m}"
    gpu, absolute = factor_checks("tall", ref, dA.cpu().numpy(), alpha.cpu().numpy(), note)   # V and R of both panels
    check(where, ref, gpu, ref.e64, absolute, note)
    b = torch.from_numpy(ref.b).to(DEV)
    x = D.ldiv(D.DistributedHouseholderQRStruct(dA, alpha, h), b).cpu().numpy()
    check(where, ref, {"x": nrm(x - ref.x_e) / nrm(ref.x_e)}, {"x": nrm(ref.x64 - ref.x_e) / nrm(ref.x_e)}, note=note)
    c = F.rhs(n, 1, seed=3, cplx=True)
    _, y_e = AO.adj_ext(ref.A, c)
    y64 = AO.np_solve_adj_c(ref.H64, ref.a64, c)
    del ref.H64
    y = D.ldiv_adjoint(D.DistributedHouseholderQRStruct(dA, alpha, h), torch.from_numpy(c).to(DEV)).cpu().numpy()
    check(where + " solve_adj", ref, {"x": nrm(y - y_e) / nrm(y_e)}, {"x": nrm(y64 - y_e) / nrm(y_e)}, note=note)
    floor = FLOOR_EPS * EPS * np.sqrt(m)
    o = orth(D.form_q(dA, handle=h))
    assert o <= C_REL * floor, f"form_q: max |Q^H Q - I| = {o:.3e} > {C_REL} x floor {floor:.1e}; {where}"


def test_large_two_panels_and_backward_error(D, h, coracle, oracle):
    # 16384 x 2048: columns 64..127 (the second panel) have been through one real-view update before their panel runs
    m, n = 16384, 2048
    ref = Ref(coracle, oracle, "normal", m, n, k=128, cplx=True, solve=False)
    ref.check_oracles_agree()
    dA, alpha, note = factor(D, ref.A, h)
    H, al = dA[:, :128].cpu().numpy(), alpha[:128].cpu().numpy()
    gpu, absolute = factor_checks("large", ref, H, al, note)
    check(f"{m}x{n} first 128 columns", ref, gpu, ref.e64, absolute, note)
    del H
    bwd = backward_error(ref.A, dA.cpu().numpy(), alpha.cpu().numpy())
    assert bwd < 1e-13, f"max_j ||(QR - A)[:, j]|| / ||A[:, j]|| = {bwd:.3e} over all {n} columns; {note}"


# ---------------------------------------------------------------------------------------------------------------------
# bits: the CTA-pair walk of k_gemm_cvy_p over odd column-tile counts
# ---------------------------------------------------------------------------------------------------------------------
def test_bitwise_across_cvy_persist_and_runs(D, h):
    m, n, k = 1000, 321, 65
    A0 = F.make_complex("centered", m, n)
    B0 = torch.from_numpy(F.rhs(m, k, cplx=True)).to(DEV)
    C0 = torch.from_numpy(np.asfortranarray(F.rhs(n, k, seed=1, cplx=True))).to(DEV)
    digests = {}
    for persist in (0, 1, 3, 4, 7):
        for run in (0, 1):
            with options(h, cvy_persist=persist):
                dA, alpha, _ = factor(D, A0, h)
                Bq = D.to_colmajor(B0, DEV)
                D.apply_qt_(Bq, dA, handle=h)
                Q = D.form_q(dA, handle=h)
                Y = D.ldiv_adjoint(D.DistributedHouseholderQRStruct(dA, alpha, h), C0)
                torch.cuda.synchronize()
            got = {"qr_c64": digest(dA.cpu().numpy(), alpha.cpu().numpy()), "apply_qt_c64": digest(Bq.cpu().numpy()),
                   "form_q_c64": digest(Q.cpu().numpy()), "solve_adj_c64": digest(Y.cpu().numpy())}
            for name, d in got.items():
                first = digests.setdefault(name, (persist, run, d))
                assert d == first[2], f"{name} with cvy_persist = {persist} (run {run}) is not bitwise equal to " \
                                      f"cvy_persist = {first[0]} (run {first[1]})"
