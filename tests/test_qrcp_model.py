"""The numpy restatement of the pivoted factorisation (tests/qrcp_model.py) against LAPACK dgeqp3 on the CPU.

On inputs whose pivots are separated (the chosen norm beats the runner-up by a relative gap >= 1e-5 at every step of LAPACK's
own factorisation) the in-place renorm, the panel width and the summation order cannot change a pivot, so the permutation must be
LAPACK's and R must agree to rounding.  normal and uniform get down to gaps of 1e-6 and kahan is all ties, so pivot identity is not
demanded for them.
"""
import numpy as np
import pytest

import matrix_families as F
import qrcp_model as M

SEPARATED = ("colscale", "graded6", "graded12", "rowscale")


@pytest.mark.parametrize("shape", [(2048, 256), (600, 200)])
@pytest.mark.parametrize("family", SEPARATED)
def test_model_matches_dgeqp3(family, shape):
    m, n = shape
    A = F.make(family, m, n)
    Hl, al, pl = M.dgeqp3_refformat(A)
    Rl = M.form_r(Hl, al)
    assert M.pivot_gap(Rl) >= 1e-5, "precondition: LAPACK's pivots are separated"
    H, a, p, _ = M.qrcp_model(A)
    assert np.array_equal(p, pl)
    cn = np.linalg.norm(A[:, p], axis=0)
    err = (np.abs(M.form_r(H, a) - Rl) / cn).max(0)
    assert err.max() < 1e-13, f"worst column {int(err.argmax())}: {err.max():.2e}"


def _qr_residual(A, H, alpha):
    m, n = A.shape
    R = np.zeros((m, n))
    R[:n] = M.form_r(H, alpha)
    for j in range(n - 1, -1, -1):
        v = H[j:, j]
        R[j:] -= np.outer(v, v @ R[j:])
    return float((np.linalg.norm(R - A, axis=0) / np.linalg.norm(A, axis=0)).max())


@pytest.mark.parametrize("shape", [(700, 96), (300, 200)])
def test_model_nearly_parallel_renorms(shape):
    m, n = shape
    A = M.nearly_parallel(m, n)
    H, a, p, renorms = M.qrcp_model(A)
    assert renorms >= 1
    assert sorted(p) == list(range(n))
    assert _qr_residual(A[:, p], H, a) < 1e-13
    # the pivot invariant: alpha_k^2 >= (1 - 1e-6) max_{c > k} ||R[k:c+1, c]||^2 while alpha_k is above the noise
    R = M.form_r(H, a)
    tail = np.sqrt(np.cumsum((R * R)[::-1], axis=0)[::-1])
    for k in range(n - 1):
        if abs(a[k]) >= 1e-8 * abs(a[0]):
            assert a[k] ** 2 >= (1 - 1e-6) * tail[k, k + 1:].max() ** 2, k


def test_model_zero_handling():
    A = F.make("zerocol_narrow", 300, 80)
    z = F.zero_column("zerocol_narrow", 80)
    H, a, p, _ = M.qrcp_model(A)
    assert np.isfinite(H).all() and np.isfinite(a).all()
    assert p[-1] == z and a[-1] == 0.0 and not H[79:, 79].any()
    H, a, p, _ = M.qrcp_model(np.zeros((50, 40), order="F"))
    assert not H.any() and not a.any() and np.array_equal(p, np.arange(40))
