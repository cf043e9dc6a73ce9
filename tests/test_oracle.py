"""Pins the CPU oracle (oracle/) — the checker the GPU parity tests rely on.

The reference holds no golden vectors; what its tests DO pin are properties (test/runtests.jl:51,62,81:
normal-equation residual < 8x LAPACK's; test/partialdot.jl:15-19: partialdot ~ dot on every suffix).
Those properties, the committed fixtures and LAPACK are checked here, on the reference's own sizes."""
import glob
import os

import numpy as np
import pytest

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "qr_*.npz")))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_c_oracle_matches_golden(path, oracle, coracle):
    g = np.load(path)
    A, b = g["A"], g["b"]
    H = np.asfortranarray(A.copy())
    H, alpha = coracle.qr(H)
    assert np.abs(H - g["H"]).max() < 1e-13
    assert np.abs(alpha - g["alpha"]).max() < 1e-13 * np.abs(g["alpha"]).max() + 1e-15
    assert np.abs(coracle.apply_qt(H, b) - g["qtb"]).max() < 1e-13
    assert np.abs(coracle.ldiv(H, alpha, b) - g["x"]).max() < 1e-10 * max(1.0, np.abs(g["x"]).max())


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_numpy_twin_matches_golden(path, oracle):
    g = np.load(path)
    H, alpha = oracle.np_qr(g["A"])
    assert np.array_equal(H, g["H"]) and np.array_equal(alpha, g["alpha"])
    assert np.allclose(oracle.np_ldiv(H, alpha, g["b"]), g["x"], rtol=1e-12, atol=1e-14)


def test_generator_c_equals_numpy(oracle, coracle):
    assert np.array_equal(coracle.fill_uniform(5, 33, 17, 2, 9), oracle.np_uniform(5, 33, 17, 2, 9))
    a = oracle.np_uniform(0, 1000, 8)
    assert 0.0 <= a.min() and a.max() < 1.0 and abs(a.mean() - 0.5) < 0.02


def test_alphafactor(oracle, coracle):
    # S:8: -sign(x), including sign(0) == 0
    for x in (2.5, -3.0, 0.0):
        assert coracle.alphafactor(x) == oracle.np_alphafactor(x) == -np.sign(x)


def test_partialdot_suffixes(oracle, coracle):
    # test/partialdot.jl:11-22 (real analogue): N = 1..20, every suffix, vs dot
    rng = np.random.default_rng(0)
    for N in range(1, 21):
        a, b = rng.random(N), rng.random(N)
        for i in range(N):
            ref = float(np.dot(a[i:], b[i:]))
            assert coracle.partialdot(a, b, i, N) == pytest.approx(ref, rel=1e-14)
            assert oracle.np_partialdot(a, b, i, N) == pytest.approx(ref, rel=1e-14)


# test/runtests.jl:42 sizes (m = 1.1 n); the two largest are exercised on the GPU side only
@pytest.mark.parametrize("mn", [(110, 100), (220, 200), (440, 400), (880, 800), (1100, 1000)])
def test_reference_property_normal_equations(mn, oracle, coracle):
    m, n = mn
    A = coracle.fill_uniform(0, m, n)
    b = oracle.np_uniform(1, m, 1)[:, 0].copy()
    x1 = oracle.lapack_lstsq(A, b)                                  # T:49
    stdliberr = oracle.normal_eq_residual(A, x1, b)                 # T:51
    H = A.copy(order="F")
    H, alpha = coracle.qr(H)                                        # T:59
    x2 = coracle.ldiv(H, alpha, b)
    assert oracle.normal_eq_residual(A, x2, b) < 8 * stdliberr      # T:62
    assert oracle.qr_residual(A, H, alpha) < 1e-13                  # BASELINE metric


@pytest.mark.parametrize("mn", [(110, 100), (1024, 128), (513, 200)])
def test_storage_format_equals_lapack(mn, oracle, coracle):
    # SURVEY App. A: alpha = diag(R), triu(H,1) = triu(R,1), v_ref = -sign(alpha) sqrt(tau) [1; v_lapack]
    m, n = mn
    A = coracle.fill_uniform(2, m, n)
    H = A.copy(order="F")
    H, alpha = coracle.qr(H)
    Hl, al = oracle.lapack_qr_refformat(A)
    assert np.abs(H - Hl).max() < 1e-12 and np.abs(alpha - al).max() < 1e-12
    # |v_j|^2 == 2 (S:131-135)
    for j in (0, n // 2, n - 1):
        assert abs(np.dot(H[j:, j], H[j:, j]) - 2.0) < 1e-13


@pytest.mark.parametrize("P", [1, 2, 3, 4])
def test_column_blocks_equal_single_block(P, oracle, coracle):
    # qr!(A::DArray) (S:115-119) == qr!(A::Matrix): every dot is rank-local (S:198-213)
    m, n = 300, 103                                        # n not divisible by P on purpose
    A = coracle.fill_uniform(4, m, n)
    b = oracle.np_uniform(5, m, 1)[:, 0].copy()
    H = A.copy(order="F")
    H, alpha = coracle.qr(H)
    bounds = [n * p // P for p in range(P + 1)]
    blocks = [np.asfortranarray(A[:, bounds[p]:bounds[p + 1]]) for p in range(P)]
    alb = coracle.qr_blocks(m, n, blocks, bounds[:-1])
    assert np.array_equal(np.hstack(blocks), H) and np.array_equal(alb, alpha)
    xb = coracle.solve_blocks(m, n, blocks, bounds[:-1], alb, b)
    assert np.allclose(xb, coracle.ldiv(H, alpha, b), rtol=1e-12, atol=1e-14)


def test_threads_do_not_change_result(coracle):
    A = coracle.fill_uniform(6, 200, 64)
    H1 = A.copy(order="F"); H8 = A.copy(order="F")
    _, a1 = coracle.qr(H1, nthreads=1)
    _, a8 = coracle.qr(H8, nthreads=8)
    assert np.array_equal(H1, H8) and np.array_equal(a1, a8)


def test_edge_cases_match_reference_behaviour(oracle, coracle):
    # n == 0 and m == n are accepted; a zero column gives f = Inf -> NaN (S:131), not an error
    H, a = coracle.qr(np.zeros((5, 0), order="F"))
    assert a.shape == (0,)
    A = coracle.fill_uniform(7, 16, 16)
    H = A.copy(order="F"); H, a = coracle.qr(H)
    assert oracle.qr_residual(A, H, a) < 1e-13
    Z = np.zeros((8, 3), order="F"); Z[:, 1] = 1.0
    with np.errstate(all="ignore"):
        Hz, az = coracle.qr(Z.copy(order="F"))
    assert np.isnan(Hz).any()


def test_qr_steps_prefix(coracle):
    # the bounded-sample entry used by bench.py's cpu_baseline runs the first j column steps of S:127
    A = coracle.fill_uniform(8, 256, 64)
    full = A.copy(order="F"); _, afull = coracle.qr(full)
    part = A.copy(order="F"); apart, fl = coracle.qr_steps(part, 10)
    assert np.array_equal(apart[:10], afull[:10]) and np.array_equal(part[:, :10], full[:, :10]) and fl > 0


# ---- ComplexF64 restatement (SURVEY 8f "next": oracle first) ----------------------------------------------------------
def _complex_matrix(oracle, seed, m, n):
    return (oracle.np_uniform(seed, m, n) - 0.5) + 1j * (oracle.np_uniform(seed + 100, m, n) - 0.5)


@pytest.mark.parametrize("m,n", [(110, 100), (300, 37), (64, 64)])
def test_complex_restatement_reconstructs_and_solves(oracle, m, n):
    A = _complex_matrix(oracle, 5, m, n)
    H, alpha = oracle.np_qr_c(A)
    # reflectors are scaled to |v|^2 = 2 (H_j = I - v v^H is unitary) and |alpha_j| is the column norm at step j
    for j in range(n):
        assert abs(np.vdot(H[j:, j], H[j:, j]).real - 2.0) < 1e-12
    assert np.linalg.norm(oracle.reconstruct_c(H, alpha) - A) / np.linalg.norm(A) < 1e-13
    # the reference's test property (T:51/62/81): normal-equation residual within 8x of LAPACK's least-squares solve
    b = _complex_matrix(oracle, 9, m, 1)[:, 0]
    x = oracle.np_ldiv_c(H, alpha, b)
    xl = np.linalg.lstsq(A, b, rcond=None)[0]
    ne = lambda z: np.linalg.norm(A.conj().T @ (A @ z - b))
    assert ne(x) < 8 * max(ne(xl), 1e-13 * np.linalg.norm(A) ** 2 * np.linalg.norm(xl))
    assert np.abs(x - xl).max() < 1e-9 * np.abs(xl).max()


def test_complex_restatement_against_lapack_zgeqrf(oracle):
    # QR is unique up to a unitary diagonal: row j of the reference's R is LAPACK's row j times the phase alpha_j / beta_j,
    # and |alpha_j| = |R_lapack[j, j]|
    from scipy.linalg import lapack
    A = _complex_matrix(oracle, 11, 200, 48)
    H, alpha = oracle.np_qr_c(A)
    qr, tau, _, info = lapack.zgeqrf(np.asfortranarray(A))
    assert info == 0
    Rl = np.triu(qr[:48])
    Rr = np.triu(H[:48], 1) + np.diag(alpha)
    phase = alpha / np.diag(Rl)
    assert np.abs(np.abs(phase) - 1.0).max() < 1e-12
    assert np.abs(Rr - phase[:, None] * Rl).max() < 1e-11 * np.abs(Rl).max()


def test_complex_alphafactor_and_partialdot(oracle):
    assert oracle.np_alphafactor_c(0.0) == -1.0                                  # angle(0) = 0 (S:9), unlike sign(0) = 0 (S:8)
    z = 3.0 - 4.0j
    assert abs(oracle.np_alphafactor_c(z) + z / abs(z)) < 1e-15
    a = _complex_matrix(oracle, 1, 50, 1)[:, 0]
    b = _complex_matrix(oracle, 2, 50, 1)[:, 0]
    for i0 in (0, 7, 49):                                                        # every suffix, test/partialdot.jl:11-22
        assert abs(oracle.np_partialdot_c(a, b, i0, 50) - np.sum(np.conj(a[i0:]) * b[i0:])) < 1e-13


# ---- extended-precision reference (the same recurrences in long double) -----------------------------------------------
def test_ext_has_extended_significand(coracle):
    # 64 bits on x86-64 (x87 extended), 113 on aarch64 (software quad): either is far enough beyond double's 53
    assert coracle.ext_mant_dig() >= 64


@pytest.mark.parametrize("mn", [(110, 100), (1024, 128), (513, 200)])
def test_ext_storage_format_equals_lapack(mn, oracle, coracle):
    m, n = mn
    A = coracle.fill_uniform(2, m, n)
    He, ae = coracle.qr_ext(A)
    Hl, al = oracle.lapack_qr_refformat(A)
    assert np.abs(He - Hl).max() < 1e-12 and np.abs(ae - al).max() < 1e-12
    b = oracle.np_uniform(3, m, 1)[:, 0].copy()
    _, _, qtb, qb, x = coracle.qr_ext(A, b, want_qb=True)
    assert np.abs(x[:, 0] - oracle.lapack_lstsq(A, b)).max() < 1e-9 * np.abs(x).max()
    assert np.abs(qtb[:, 0] - coracle.apply_qt(coracle.qr(A.copy(order="F"))[0], b)).max() < 1e-13 * np.sqrt(m)
    # Qb applies the same reflectors in reverse order: Q(Q'b) = b
    w = qtb[:, 0].copy()
    for j in range(n - 1, -1, -1):
        w[j:] -= He[j:, j] * (He[j:, j] @ w[j:])
    assert np.abs(w - b).max() < 1e-13 * np.sqrt(m)
    assert np.abs(np.linalg.norm(qb[:, 0]) - np.linalg.norm(b)) < 1e-13 * np.linalg.norm(b)


def test_ext_is_independent_of_thread_count(coracle):
    A = coracle.fill_uniform(6, 300, 97)
    b = np.asfortranarray(coracle.fill_uniform(7, 300, 2))
    r1 = coracle.qr_ext(A, b, nthreads=1, want_qb=True)
    r5 = coracle.qr_ext(A, b, nthreads=5, want_qb=True)
    for u, v in zip(r1, r5):
        assert np.array_equal(u, v)
    c1 = coracle.qr_ext_c(A + 1j * A[::-1], b[:, 0] + 0j, nthreads=1)
    c3 = coracle.qr_ext_c(A + 1j * A[::-1], b[:, 0] + 0j, nthreads=3)
    for u, v in zip(c1, c3):
        assert np.array_equal(u, v)


def test_ext_mirrors_zero_column_and_zero_pivot(oracle, coracle):
    # the same recurrences, so the same divergences: a zero column gives NaN from that column on (S:131), an exactly zero
    # pivot gives alpha = 0 (S:8)
    Z = coracle.fill_uniform(8, 40, 6)
    Z[:, 2] = 0.0
    with np.errstate(all="ignore"):
        H, a = coracle.qr(Z.copy(order="F"))
        He, ae = coracle.qr_ext(Z)
    assert np.array_equal(np.isnan(He), np.isnan(H)) and np.array_equal(np.isnan(ae), np.isnan(a))
    assert np.isnan(He[2:, 2]).all() and np.isfinite(He[:, :2]).all()
    P = coracle.fill_uniform(9, 40, 6)
    P[0, 0] = 0.0
    assert coracle.qr_ext(P)[1][0] == 0.0


SIGNED_ZERO_PIVOTS = [(complex(0.0, 0.0), -1.0), (complex(0.0, -0.0), -1.0),
                      (complex(-0.0, 0.0), 1.0 - 1.2246467991473532e-16j), (complex(-0.0, -0.0), 1.0 + 1.2246467991473532e-16j)]


@pytest.mark.parametrize("x0,af", SIGNED_ZERO_PIVOTS, ids=["+0+0i", "+0-0i", "-0+0i", "-0-0i"])
def test_complex_zero_pivot_follows_the_signs_of_its_zeros(oracle, coracle, x0, af):
    # alphafactor(x::Complex) = -exp(im * angle(x)) (S:9) and angle = atan2(imag, real) sees the sign of a zero: angle(-0 +- 0i)
    # = +-pi.  The numpy oracle, the long double oracle (qr_ext_c and the adjoint reference) and dhqr_b200.alphafactor agree
    import adjoint_oracle as AO
    import dhqr_b200
    assert oracle.np_alphafactor_c(x0) == af and dhqr_b200.alphafactor(x0) == af
    A = np.asfortranarray(np.array([[x0, 1.0], [3.0 - 4.0j, 2.0j], [0.0, 1.0 + 1.0j]], dtype=np.complex128))
    s = 5.0
    Hn, an = oracle.np_qr_c(A)
    He, ae = coracle.qr_ext_c(A)
    assert an[0] == s * af and ae[0] == s * af
    assert np.abs(He - Hn).max() < 1e-15 and np.abs(ae - an).max() < 1e-14
    assert abs(Hn[0, 0] - (x0 - s * af) / s) < 1e-16                                     # f = 1 / s: |x0| = 0 (S:131)
    # adj_ext factors in long double with the same convention: z_0 = c_0 / conj(alpha_0)
    z, _ = AO.adj_ext(A, np.array([1.0 + 0j, 0.0]))
    assert abs(z[0] - 1.0 / np.conj(s * af)) < 1e-16


@pytest.mark.parametrize("family,h_err,a_err", [("uniform", 2.5e-14, 1.6e-16), ("normal", 1.3e-14, 3.5e-16),
                                                ("graded6", 5.4e-12, 2.6e-12), ("graded12", 3.5e-6, 1.2e-6)])
def test_fp64_oracle_forward_error_against_ext(family, h_err, a_err, oracle, coracle):
    # pins the yardstick: at 2048 x 512 the fp64 oracle sits where kappa * eps puts it, and the extended reference is far
    # enough beyond it to measure that (a lower bound too: an "extended" reference that rounded like double would give 0)
    import matrix_families as F
    A = F.make(family, 2048, 512, 0)
    He, ae = coracle.qr_ext(A)
    H, a = coracle.qr(A.copy(order="F"))
    eh = np.abs(H - He).max()
    ea = (np.abs(a - ae) / np.abs(ae)).max()
    assert h_err / 8 < eh < h_err * 8, eh
    assert a_err / 8 < ea < a_err * 8, ea


def test_ext_complex_matches_numpy_twin_and_lstsq(oracle, coracle):
    A = _complex_matrix(oracle, 13, 300, 37)
    b = _complex_matrix(oracle, 14, 300, 1)[:, 0]
    He, ae, qtb, x = coracle.qr_ext_c(A, b)
    Hn, an = oracle.np_qr_c(A)
    assert np.abs(He - Hn).max() < 1e-13 and np.abs(ae - an).max() < 1e-13 * np.abs(an).max()
    assert np.abs(qtb[:, 0] - oracle.np_apply_qt_c(Hn, b)).max() < 1e-13 * np.sqrt(300)
    xl = np.linalg.lstsq(A, b, rcond=None)[0]
    assert np.abs(x[:, 0] - xl).max() < 1e-12 * np.abs(xl).max()
    assert np.array_equal(coracle.ldiv_ext_c(A, b), x[:, 0])
