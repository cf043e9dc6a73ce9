"""The CTA pairs of k_gemm_cvy_p: both CTAs of a 2-CTA cluster run the same row tile on adjacent column tiles and multicast
one V slice each to both.  Cases aimed at the pairing:

  - odd column-tile counts (1, 3 and 5 tiles, and a ragged 2-tile width), where rank 1 of the last column pair has no tile and
    must only keep the shared V ring turning, on the bulk (even lda) and generic (odd lda) C paths;
  - walk lengths (cvy_persist) that split the pair-tiles unevenly, including phantom tiles in the middle of a pair's walk:
    every walk length gives bitwise the same result;
  - fewer than 128 rows (one row tile, four k-stages) and row_lo at or past 128 (dead row tiles in the walk);
  - qr_ where every paired trailing update has an odd number of 64-column tiles, against the oracle and the narrow chain, and
    bitwise across walk lengths.

Block-reflector cases go through dhqr_k_block_reflector_f64 and are checked against torch fp64 (relative error <= 1e-13), with
NaN in the lda padding rows and the rows above row_lo bitwise untouched."""
import numpy as np
import pytest
import torch

from test_gpu_cvy_stream import Case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture
def h(D):
    hd = D.default_handle(0)
    persist = hd.get_option("cvy_persist")
    yield hd
    hd.set_option("cvy_persist", persist)


@pytest.mark.parametrize("ncols", [1, 65, 192, 5 * 64 - 7])
@pytest.mark.parametrize("lda_extra", [0, 1])   # rows even: lda = rows takes the bulk C path, rows + 1 the generic one
def test_odd_column_tile_counts(D, h, ncols, lda_extra):
    rows = 1000
    cs = Case(D, rows, 0, ncols, seed=11)
    lda = rows + lda_extra
    where = f"rows {rows}, ncols {ncols}, lda {lda}"
    buf, dC = cs.run(D, h, lda)
    cs.check(buf, dC, lda, 0, where)
    _, dC2 = cs.run(D, h, lda)
    assert torch.equal(dC, dC2), f"two runs differ; {where}"


@pytest.mark.parametrize("rows,ncols", [(4099, 5 * 64 - 7), (1000, 192), (129, 65), (100, 1)])
def test_pair_walk_lengths_bitwise_equal(D, h, rows, ncols):
    cs = Case(D, rows, 0, ncols, seed=12)
    lda = rows + 1
    first = None
    for persist in (0, 1, 3, 4, 7):
        h.set_option("cvy_persist", persist)
        buf, dC = cs.run(D, h, lda)
        where = f"rows {rows}, ncols {ncols}, lda {lda}, cvy_persist {persist}"
        if first is None:
            cs.check(buf, dC, lda, 0, where)
            first = dC.clone()
        else:
            assert torch.equal(dC, first), f"differs from cvy_persist 0; {where}"
        del buf, dC


@pytest.mark.parametrize("rows,row_lo", [(1, 0), (50, 3), (127, 0), (300, 128), (1000, 200), (1000, 640)])
def test_short_rows_and_high_row_lo(D, h, rows, row_lo):
    for ncols in (64, 192):
        cs = Case(D, rows, row_lo, ncols, seed=13)
        for lda in (rows + (rows & 1), rows + 1 - (rows & 1)):   # one even and one odd leading dimension
            where = f"rows {rows}, row_lo {row_lo}, ncols {ncols}, lda {lda}"
            buf, dC = cs.run(D, h, lda)
            cs.check(buf, dC, lda, 0, where)


def qr_run(D, dev, A0, **opts):
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


def test_qr_pairs_with_odd_trailing_tile_counts(D, oracle, coracle):
    # n = 832: the pairs (0, 1), (2, 3) and (4, 5) leave 576, 320 and 64 trailing columns, 9, 5 and 1 column tiles
    dev = torch.device("cuda:0")
    m, n = 2999, 832
    A0 = coracle.fill_uniform(21, m, n)
    h = D.default_handle(0)
    p0 = h.get_option("pair_units")
    Hx, ax = qr_run(D, dev, A0)
    assert h.get_option("pair_units") > p0
    Hn, an = qr_run(D, dev, A0, wide_panel=0)
    assert oracle.qr_residual(A0, np.asfortranarray(Hx), ax) < 1e-13
    assert np.abs(Hx - Hn).max() < 1e-10
    assert np.abs(ax - an).max() < 1e-12 * np.abs(an).max()
    for persist in (0, 1, 3, 7):
        Hp, ap = qr_run(D, dev, A0, cvy_persist=persist)
        assert np.array_equal(Hp, Hx) and np.array_equal(ap, ax), f"cvy_persist {persist} differs from the default walk"
