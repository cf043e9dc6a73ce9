"""The numpy restatement of the ComplexF64 pivoted factorisation (qrcp_c_model) against LAPACK zgeqp3, without a GPU.

The model is what the device kernels of dhqr_qrcp_c64 compute, panel by panel with the in-panel renorm; here it is held to
LAPACK: the same pivots on complex families whose column norms are well separated, the same R up to the phases of its diagonal
(zgeqp3 makes the diagonal real, the library's alpha = -exp(i angle(x0)) ||x|| does not), A[:, p] = Q R from the stored
reflectors, renorms on nearly parallel complex columns, and the signed-zero pivots of k_house1_c.
"""
import numpy as np
import pytest

import matrix_families as F
import qrcp_c_model as M

SEPARATED = ("colscale", "graded6", "graded12", "rowscale")


def rel_cols(X, Y):
    """max over columns of ||X[:, c] - Y[:, c]|| / ||Y[:, c]||."""
    return float((np.linalg.norm(X - Y, axis=0) / np.linalg.norm(Y, axis=0)).max())


def scaled(A):
    """A with each column scaled by a power of two near its norm (exact), so 1e+-120 columns compare on one scale."""
    cn = np.linalg.norm(A, axis=0)
    return A / np.ldexp(1.0, np.round(np.log2(np.where(cn > 0, cn, 1.0))).astype(int))


@pytest.mark.parametrize("family", SEPARATED)
def test_model_matches_zgeqp3(family):
    m, n = 300, 96
    A0 = F.make_complex(family, m, n)
    H, alpha, p, _ = M.qrcp_c_model(A0)
    Rl, pl = M.zgeqp3_refformat(A0)
    assert np.array_equal(p, pl)
    R = M.form_r(H, alpha)
    d = alpha / np.diag(Rl)
    d = d / np.abs(d)                                                  # D is unitary
    cn = np.linalg.norm(A0[:, p], axis=0)
    assert float((np.abs(np.abs(alpha) - np.abs(np.diag(Rl))) / cn).max()) < 1e-13
    assert float((np.abs(R - d[:, None] * Rl) / cn).max()) < 1e-13     # R = D R_lapack, column-relative


@pytest.mark.parametrize("family", ("normal", "graded6", "colscale", "imag", "kahan"))
@pytest.mark.parametrize("m,n", [(200, 70), (96, 96), (130, 33)])
def test_model_reconstructs(family, m, n):
    A0 = F.make_complex(family, m, n)
    H, alpha, p, _ = M.qrcp_c_model(A0)
    assert sorted(p) == list(range(n))
    assert np.abs((np.abs(np.tril(H)) ** 2).sum(0) - 2.0).max() < 1e-13   # |v|^2 = 2
    Q = M.form_q(H)
    assert rel_cols(scaled(Q @ M.form_r(H, alpha)), scaled(A0[:, p])) < 1e-13
    R = M.form_r(H, alpha)
    tail = np.sqrt(np.cumsum((np.abs(R) ** 2)[::-1], axis=0)[::-1])
    for k in range(n - 1):                                             # the pivot invariant
        if abs(alpha[k]) >= 1e-8 * abs(alpha[0]):
            assert abs(alpha[k]) ** 2 >= (1 - 1e-6) * tail[k, k + 1:].max() ** 2


def test_model_renorms():
    A0 = M.nearly_parallel(400, 64)
    H, alpha, p, renorms = M.qrcp_c_model(A0)
    assert renorms >= 1
    Rl, pl = M.zgeqp3_refformat(A0)
    # the columns are nearly parallel, so the pivots past the first are decided by 1e-10 perturbations: compare |diag(R)| only
    assert np.abs(np.abs(alpha[:8]) - np.abs(np.diag(Rl))[:8]).max() <= 1e-6 * abs(alpha[0])
    Q = M.form_q(H)
    assert rel_cols(Q @ M.form_r(H, alpha), A0[:, p]) < 1e-13


@pytest.mark.parametrize("x0", [complex(0.0, 0.0), complex(0.0, -0.0), complex(-0.0, 0.0), complex(-0.0, -0.0), 3 - 4j])
def test_house_signed_zero_pivots(x0):
    x = np.array([x0, 1 + 2j, -0.5j], dtype=np.complex128)
    al, v = M.house_c(x)
    s = np.linalg.norm(x)
    ref = -np.exp(1j * np.angle(x0)) * s                               # numpy's angle sees the signs of a zero
    assert al.real == pytest.approx(ref.real, rel=1e-15, abs=1e-300) and al.imag == pytest.approx(ref.imag, rel=1e-15, abs=1e-300)
    assert np.signbit(al.real) == np.signbit(ref.real)                 # a zero imaginary part may carry either sign
    assert abs(np.vdot(v, v) - 2.0) < 1e-15
    Hx = x - v * np.vdot(v, x)
    assert abs(Hx[0] - al) < 1e-14 * s and np.abs(Hx[1:]).max() < 1e-14 * s


def test_model_zero_matrix_and_zero_column():
    H, alpha, p, _ = M.qrcp_c_model(np.zeros((50, 40), dtype=np.complex128, order="F"))
    assert not H.any() and not alpha.any() and np.array_equal(p, np.arange(40))
    A0 = F.make_complex("zerocol_mid", 200, 70)
    H, alpha, p, _ = M.qrcp_c_model(A0)
    assert p[-1] == F.zero_column("zerocol_mid", 70) and alpha[-1] == 0 and not H[69:, 69].any()
