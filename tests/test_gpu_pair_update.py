"""GPU tests of the paired trailing update: two 128-column panels of the wide chain applied as one 256-wide block reflector
(apply_pair: W_a, W_b, G = V_b' V_a, k_ymake2, then k_gemm_cvy_p with 8 k-stages).  Same tolerances as
tests/test_gpu_wide.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL_H, TOL_RES = 1e-10, 1e-13


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def run(D, dev, A0, **opts):
    h = D.default_handle(0)
    old = {k: h.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            h.set_option(k, v)
        A = D.to_colmajor(A0, dev)
        H = D.qr_(A)
        torch.cuda.synchronize()
        return A.cpu().numpy(), H.α.cpu().numpy()
    finally:
        for k, v in old.items():
            h.set_option(k, v)


def test_pair_counter_at_the_bench_shape(D, dev):
    # 32768 x 4096, nb = 128: 32 wide panels, paired into 16 units
    h = D.default_handle(0)
    m, n = 32768, 4096
    A = D.colmajor_empty(m, n, dev)
    D.fill_uniform_(A, 0)
    p0, w0 = h.get_option("pair_units"), h.get_option("wide_panels")
    D.qr_(A)
    torch.cuda.synchronize()
    assert h.get_option("pair_units") - p0 == 16
    assert h.get_option("wide_panels") - w0 == 32


@pytest.mark.parametrize("mn", [(3000, 640), (2050, 1000), (1537, 777), (4096, 1024)])
@pytest.mark.parametrize("lookahead", [1, 0])
def test_pairs_against_oracle_and_narrow_chain(D, dev, oracle, coracle, mn, lookahead):
    # even and odd panel counts, ragged last panels (a single unit), odd m; the look-ahead and the serial schedule
    m, n = mn
    A0 = coracle.fill_uniform(3, m, n)
    Hx, ax = run(D, dev, A0, lookahead=lookahead)
    Hn, an = run(D, dev, A0, wide_panel=0)
    assert oracle.qr_residual(A0, np.asfortranarray(Hx), ax) < TOL_RES
    assert np.abs(Hx - Hn).max() < TOL_H
    assert np.abs(ax - an).max() < 1e-12 * np.abs(an).max()


def test_pairs_bitwise_repeatable_and_walk_invariant(D, dev, coracle):
    A0 = coracle.fill_uniform(5, 4099, 1280)
    H1, a1 = run(D, dev, A0)
    H2, a2 = run(D, dev, A0)
    H3, a3 = run(D, dev, A0, cvy_persist=0)
    assert np.array_equal(H1, H2) and np.array_equal(a1, a2)
    assert np.array_equal(H1, H3) and np.array_equal(a1, a3)


@pytest.mark.parametrize("col", [100, 200, 330])
def test_restart_after_a_refused_panel_of_a_pair(D, dev, oracle, coracle, col):
    # column `col` nearly a copy of an earlier one: the wide chain refuses its panel, the first panel of pair (0, 1) (col 100),
    # its second (col 200: V_0 must reach the columns right of panel 1 before the restart) or the first of pair (2, 3) (col 330).
    # The restart must give the answer of the wide chain off.
    h = D.default_handle(0)
    m, n = 3000, 768
    A0 = coracle.fill_uniform(12, m, n)
    A0[:, col] = A0[:, col - 50] + 1e-11 * coracle.fill_uniform(13, m, 1)[:, 0]
    r0 = h.get_option("wide_redone")
    Hx, ax = run(D, dev, A0)
    assert h.get_option("wide_redone") == r0 + 1
    Hn, an = run(D, dev, A0, wide_panel=0)
    assert oracle.qr_residual(A0, np.asfortranarray(Hx), ax) < TOL_RES
    assert oracle.qr_residual(A0, np.asfortranarray(Hn), an) < TOL_RES
    assert np.abs(ax - an).max() < 1e-5 * np.abs(an).max()
    keep = (col // 128) * 128                                    # panels before the refused one: exact parity
    if keep:
        assert np.abs(Hx[:, :keep] - Hn[:, :keep]).max() < TOL_H
