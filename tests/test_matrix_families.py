"""The complex test matrices of tests/matrix_families.py (CPU only): structure, determinism and the positions of exact zeros,
which the accuracy modules rely on without looking."""
import numpy as np
import pytest

import matrix_families as F

SHAPES = [(1024, 384), (777, 321), (130, 64)]


def parts(a):
    """Real and imaginary parts of every entry, as one float64 vector."""
    return np.concatenate([a.real.ravel(), a.imag.ravel()])


@pytest.mark.parametrize("family", F.COMPLEX_ALL)
def test_complex_family_is_a_seeded_function_of_its_arguments(family):
    m, n = 260, 97
    a = F.make_complex(family, m, n)
    assert a.dtype == np.complex128 and a.shape == (m, n) and a.flags.f_contiguous
    b = F.make_complex(family, m, n)
    assert a.tobytes() == b.tobytes()                                    # the signs of zeros included
    assert F.make_complex(family, m, n, seed=1).tobytes() != a.tobytes()
    assert np.isfinite(a).all()
    if family in F.FAMILIES:                                             # a twin of a real family, not a copy of it
        assert np.abs(a.imag).max() > 0 and not np.array_equal(a.real, F.make(family, m, n))


def test_existing_complex_families_are_unchanged():
    # other modules pin numbers measured on these three; their draws must not move
    rng = np.random.default_rng([ord(c) for c in "ccentered"] + [50, 20, 0])
    want = (rng.random((50, 20)) - 0.5) + 1j * (rng.random((50, 20)) - 0.5)
    assert np.array_equal(F.make_complex("centered", 50, 20), want)
    assert F.COMPLEX_FAMILIES == ("centered", "graded6", "colscale")


@pytest.mark.parametrize("m,n", SHAPES)
def test_complex_structure(m, n):
    sv = lambda a: np.linalg.svd(a, compute_uv=False)
    tri = F.make_complex("triangular", m, n)
    assert not np.tril(tri[:n], -1).any() and not tri[n:].any() and (np.diag(tri) != 0).all()
    zr = F.make_complex("zerorows", m, n)
    z = F.zero_rows(m, n)
    assert not zr[m - z:].any() and (zr[:m - z] != 0).all()
    # kahan: the real Kahan matrix with unit-modulus row and column phases, so the same singular values
    k = F.make_complex("kahan", m, n)
    kr = F.make("kahan", m, n)
    assert np.allclose(np.abs(k), np.abs(kr), rtol=1e-15, atol=0)
    assert np.allclose(sv(k), sv(kr), rtol=0, atol=1e-13 * sv(kr)[0])
    assert np.angle(k[:n][np.abs(kr[:n]) > 0]).std() > 1.5                # phases spread over (-pi, pi]: std pi / sqrt(3)
    im = F.make_complex("imag", m, n)
    assert not np.signbit(im.real).any() and not im.real.any() and (im.imag != 0).all()
    for fam, lo, hi in (("tiny", 1e-160, 1e-148), ("huge", 1e140, 1e152)):
        a = np.abs(F.make_complex(fam, m, n))
        assert lo < np.median(a) < hi and np.linalg.norm(a, axis=0).max() < 1e300
    rs = F.make_complex("rowscale", m, n)
    rmax = np.abs(rs).max(1)
    assert rmax.max() / rmax.min() > 1e8
    g = F.make_complex("graded6", m, n)
    s = sv(g)
    assert 0.5e6 < s[0] / s[-1] < 2e6


@pytest.mark.parametrize("m,n", SHAPES)
def test_complex_zero_columns_sit_where_the_panels_put_them(m, n):
    cols = {}
    for fam in F.COMPLEX_NAN_FAMILIES:
        a = F.make_complex(fam, m, n)
        j = F.zero_column(fam, n)
        zero = ~np.abs(a).any(0)
        assert np.array_equal(np.nonzero(zero)[0], [j]), fam
        assert F.singular(fam, m, n)
        cols[fam] = j
    if n >= 2 * F.CPW:
        assert cols["zerocol_first"] % F.CPW == 0 and cols["zerocol_first"] > 0
        assert 0 < cols["zerocol_mid"] % F.CPW < F.CPW - 1
        assert cols["zerocol_last"] % F.CPW == F.CPW - 1 and cols["zerocol_last"] < n


@pytest.mark.parametrize("m,n", [(1024, 384), (777, 321), (128, 64)])
def test_zerolead_layout_and_its_signed_zeros(m, n):
    a = F.make_complex("zerolead", m, n)
    top = parts(a[:n])
    assert not top.any() and not np.signbit(top).any()                  # exactly +0, both parts
    d = np.diagonal(a[n:2 * n])
    assert np.array_equal(a[n:2 * n], np.diag(d)) and (np.abs(d) >= 1).all() and (np.abs(d) < 2).all()
    assert (np.abs(d.imag) > 0).any() and (np.abs(a[2 * n:]) > 0).all()
    for fam, im_sign in (("zerolead_neg", False), ("zerolead_negneg", True)):
        b = F.make_complex(fam, m, n)
        x0 = b[0, 0]
        assert x0 == 0 and np.signbit(x0.real) and np.signbit(x0.imag) == im_sign
        c = b.copy()
        c[0, 0] = 0.0                                                   # otherwise the zerolead layout: +0 on top, diag(d) below
        assert not parts(c[:n]).any() and not np.signbit(parts(c[:n])).any()
        assert np.array_equal(c[n:2 * n], np.diag(np.diagonal(c[n:2 * n])))
    with pytest.raises(ValueError):
        F.make_complex("zerolead", 2 * n - 1, n)


def test_zerolead_pivots_are_exact_zeros_in_the_oracle(oracle):
    # the property the GPU test builds on: in the reference recurrence every pivot of zerolead is an exact +0, so every
    # alpha_j = -s_j (real, negative) and v_j is 1 on its diagonal and exactly zero on rows j+1..n-1
    m, n = 200, 70
    a = F.make_complex("zerolead", m, n)
    H, alpha = oracle.np_qr_c(a)
    assert (alpha.real < 0).all() and not alpha.imag.any()
    assert np.abs(np.diagonal(H) - 1.0).max() <= np.finfo(np.float64).eps
    for j in range(n):
        assert not H[j + 1:n, j].any()


def test_complex_nan_families_give_the_oracles_nan_pattern(oracle, coracle):
    from ext_rule import Ref
    m, n = 300, 130
    for fam in F.COMPLEX_NAN_FAMILIES:
        r = Ref(coracle, oracle, fam, m, n, cplx=True)
        j = F.zero_column(fam, n)
        assert r.k == j and not r.solve
        assert np.array_equal(r.nan_cols, np.arange(n) >= j), fam
        assert np.array_equal(r.nan_alpha, np.arange(n) > j), fam
        assert r.He.shape == (m, j)
        r.check_oracles_agree()
