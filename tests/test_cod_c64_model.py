"""The long-double ComplexF64 twin of the complete orthogonal decomposition solve (cod_c_model.cod_ext_c) against numpy, without
a GPU: on exactly rank-r complex matrices it is the minimum-norm least-squares solution, numpy.linalg.lstsq's and the SVD
pseudo-inverse's, for any permutation, and at full rank it is the ordinary least-squares solution."""
import numpy as np
import pytest

import cod_c_model as CM
import qrcp_c_model as M


@pytest.mark.parametrize("r", [1, 7, 33, 64])
def test_cod_ext_c_is_the_pseudo_inverse(r):
    m, n = 160, 80
    A0 = M.low_rank(m, n, r)
    rng = np.random.default_rng([m, n, r])
    b = rng.standard_normal((m, 3)) + 1j * rng.standard_normal((m, 3))
    _, _, p, _ = M.qrcp_c_model(A0)
    x = CM.cod_ext_c(A0, p, r, b)
    xp = CM.pinv_solve_c(A0, b, r)
    xl = np.linalg.lstsq(A0, b, rcond=1e-10)[0]
    assert np.abs(x - xp).max() <= 1e-11 * np.abs(xp).max()
    assert np.abs(x - xl).max() <= 1e-11 * np.abs(xl).max()
    # any permutation gives the same minimum-norm solution on exactly rank-r input, once the first r columns span the range
    x1 = CM.cod_ext_c(A0, p[::-1].copy(), r, b[:, 0])
    assert np.abs(x1 - xp[:, 0]).max() <= 1e-9 * np.abs(xp[:, 0]).max()


def test_cod_ext_c_full_rank_is_least_squares():
    m, n = 120, 50
    rng = np.random.default_rng(5)
    A0 = rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n))
    b = rng.standard_normal(m) + 1j * rng.standard_normal(m)
    p = rng.permutation(n)
    x = CM.cod_ext_c(A0, p, n, b)
    assert np.abs(x - np.linalg.lstsq(A0, b, rcond=None)[0]).max() <= 1e-12 * np.abs(x).max()
    assert not CM.cod_ext_c(A0, p, 0, b).any()
