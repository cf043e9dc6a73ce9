"""The C path of the 128-wide block-reflector update (k_gemm_cvy_p): C tiles reach shared memory by bulk copies and leave by
bulk stores when C is 16 B aligned and ldc is even, rows outside a column's even-aligned bulk segment move by generic loads and
stores, and every other C takes the generic path.  Cases aimed at that path:

  - a C base 8 B off 16 B alignment with an even ldc (generic path with a stride that would allow bulk copies);
  - odd row_lo with ragged row counts (the odd ends of every bulk-stored segment), lda = rows and rows + 1;
  - walk lengths (cvy_persist) that do not divide the tile count, and a long walk that reuses the C buffer many times in one
    CTA: every walk length gives bitwise the same result, because a tile's arithmetic does not depend on the CTA that runs it;
  - row_lo at or past 128, so that whole row tiles are dead (no bytes to copy on the bulk path);
  - two updates of disjoint column ranges of one matrix, on two handles and two non-blocking streams at once: bitwise equal
    to the same two updates run one after the other.  A store wider than its own columns shows here only when the two
    updates happen to overlap in time, which this race-based check cannot force; the sequential runs are also compared with
    each other.

Every case goes through dhqr_k_block_reflector_f64 and is checked against torch fp64 (relative error <= 1e-13), with NaN in
the lda padding rows and the rows above row_lo bitwise untouched."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def householder_block(rows, row_lo, nbp, seed):
    """rows x nbp: reflectors with |v|^2 = 2 (or 0) on rows >= row_lo, zero above."""
    g = torch.Generator().manual_seed(seed)
    a, tau = torch.geqrf(torch.rand(rows - row_lo, nbp, dtype=torch.float64, generator=g))
    k = tau.numel()
    Vk = torch.tril(a[:, :k], -1) + torch.eye(rows - row_lo, k, dtype=torch.float64)
    V = torch.zeros(rows, nbp, dtype=torch.float64)
    V[row_lo:, :k] = Vk * tau.sqrt()
    return V


class Case:
    """V (rows x nbp) on rows >= row_lo, C0 (rows x ncols) and the torch fp64 result."""

    def __init__(self, D, rows, row_lo, ncols, nbp=128, seed=0, C0=None):
        self.rows, self.row_lo, self.ncols, self.nbp = rows, row_lo, ncols, nbp
        V = householder_block(rows, row_lo, nbp, seed=seed * 7919 + rows * 131 + row_lo)
        self.dV = D.to_colmajor(V, DEV)
        Vd = V.to(DEV)
        L = torch.eye(nbp, dtype=torch.float64, device=DEV) + torch.tril(Vd.T @ Vd, -1)
        Linv = torch.linalg.solve_triangular(L, torch.eye(nbp, dtype=torch.float64, device=DEV), upper=False)
        self.C0 = C0 if C0 is not None else torch.rand(rows, ncols, dtype=torch.float64, device=DEV,
                                                       generator=torch.Generator(device=DEV).manual_seed(seed * 1009 + ncols))
        self.Cexp = self.C0 - Vd @ (Linv @ (Vd.T @ self.C0))

    def buffer(self, lda, offset=0):
        """NaN-filled storage; C starts `offset` doubles into it with leading dimension lda."""
        buf = torch.full((offset + self.ncols * lda,), float("nan"), dtype=torch.float64, device=DEV)
        dC = buf[offset:].as_strided((self.rows, self.ncols), (1, lda))
        dC.copy_(self.C0)
        return buf, dC

    def launch(self, D, h, dC, lda, stream, col0=0, ncols=None):
        """Enqueue the update of columns [col0, col0 + ncols) of dC on `stream` (no synchronisation)."""
        ncols = self.ncols - col0 if ncols is None else ncols
        ptr = dC.data_ptr() + 8 * col0 * lda
        D._lib.call("dhqr_k_block_reflector_f64", h.raw, self.rows, self.nbp, C.c_void_p(self.dV.data_ptr()), self.rows,
                    self.row_lo, ncols, C.c_void_p(ptr), lda, None, C.c_void_p(stream.cuda_stream))

    def run(self, D, h, lda, offset=0):
        buf, dC = self.buffer(lda, offset)
        self.launch(D, h, dC, lda, torch.cuda.current_stream())
        torch.cuda.synchronize()
        return buf, dC

    def check(self, buf, dC, lda, offset, where):
        rows, ncols, row_lo = self.rows, self.ncols, self.row_lo
        if offset:
            assert torch.isnan(buf[:offset]).all(), f"storage before C written; {where}"
        if lda > rows:
            assert torch.isnan(buf[offset:].view(ncols, lda)[:, rows:]).all(), f"lda padding written; {where}"
        assert torch.equal(dC[:row_lo], self.C0[:row_lo]), f"rows above row_lo changed; {where}"
        ref = self.Cexp[row_lo:]
        err = float((dC[row_lo:] - ref).abs().max() / ref.abs().max())
        assert err < 1e-13, f"relative error {err:.2e}; {where}"


@pytest.fixture
def h(D):
    hd = D.default_handle(0)
    persist = hd.get_option("cvy_persist")
    yield hd
    hd.set_option("cvy_persist", persist)


@pytest.mark.parametrize("rows", [129, 4099])
@pytest.mark.parametrize("ncols", [65, 200])
def test_misaligned_c_even_ldc(D, h, rows, ncols):
    cs = Case(D, rows, 0, ncols, seed=1)
    lda, offset = rows + 1, 1            # even leading dimension, C base 8 B past a 16 B boundary
    buf, dC = cs.run(D, h, lda, offset)
    assert (dC.data_ptr() % 16) == 8
    where = f"rows {rows}, ncols {ncols}, lda {lda}, offset 8 B"
    cs.check(buf, dC, lda, offset, where)
    _, dC2 = cs.run(D, h, lda, offset)
    assert torch.equal(dC, dC2), f"two runs differ; {where}"


@pytest.mark.parametrize("rows", [129, 1000, 4099])
@pytest.mark.parametrize("row_lo", [1, 3, 31, 33])
def test_odd_row_lo_ragged_rows(D, h, rows, row_lo):
    for ncols in (64, 130):
        cs = Case(D, rows, row_lo, ncols, seed=2)
        for lda in (rows, rows + 1):
            where = f"rows {rows}, row_lo {row_lo}, ncols {ncols}, lda {lda}"
            buf, dC = cs.run(D, h, lda)
            cs.check(buf, dC, lda, 0, where)
            _, dC2 = cs.run(D, h, lda)
            assert torch.equal(dC, dC2), f"two runs differ; {where}"


@pytest.mark.parametrize("rows", [1000, 4099])
@pytest.mark.parametrize("row_lo", [128, 129, 256, 385])
def test_row_lo_past_whole_tiles(D, h, rows, row_lo):
    cs = Case(D, rows, row_lo, 130, seed=6)
    for lda in (rows, rows + 1):
        where = f"rows {rows}, row_lo {row_lo}, ncols 130, lda {lda}"
        buf, dC = cs.run(D, h, lda)
        cs.check(buf, dC, lda, 0, where)
        _, dC2 = cs.run(D, h, lda)
        assert torch.equal(dC, dC2), f"two runs differ; {where}"


@pytest.mark.parametrize("rows,ncols", [(4099, 200), (1000, 65), (32768, 3712)])
def test_walk_lengths_bitwise_equal(D, h, rows, ncols):
    cs = Case(D, rows, 0, ncols, seed=3)
    lda = rows + 1 if rows < 32768 else rows
    first = None
    for persist in (0, 1, 2, 3, 4, 8, 64):
        h.set_option("cvy_persist", persist)
        buf, dC = cs.run(D, h, lda)
        where = f"rows {rows}, ncols {ncols}, lda {lda}, cvy_persist {persist}"
        if first is None:
            cs.check(buf, dC, lda, 0, where)
            first = dC.clone()
        else:
            assert torch.equal(dC, first), f"differs from cvy_persist 0; {where}"
        del buf, dC


@pytest.mark.parametrize("lda_extra", [0, 2])
def test_disjoint_columns_on_two_streams(D, lda_extra):
    rows, n1, n2 = 8195, 100, 165         # n1 is not a multiple of the 64-column tile
    lda = rows + 1 + lda_extra            # even: bulk copies
    a = Case(D, rows, 5, n1 + n2, seed=4)
    b = Case(D, rows, 5, n1 + n2, seed=5, C0=a.C0)   # a second V on the same C; it updates columns [n1, n1 + n2)
    h1, h2 = D.Handle(0), D.Handle(0)   # the hook packs V into its handle's workspace: one handle runs one update at a time
    try:
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()   # non-blocking with respect to each other
        main = torch.cuda.current_stream()

        def both(concurrent):
            buf, dC = a.buffer(lda)
            s1.wait_stream(main)
            s2.wait_stream(main)
            a.launch(D, h1, dC, lda, s1, col0=0, ncols=n1)
            b.launch(D, h2, dC, lda, s1 if not concurrent else s2, col0=n1, ncols=n2)
            torch.cuda.synchronize()
            return buf, dC

        _, seq0 = both(False)                                # workspace growth happens here, not in the concurrent call
        buf_seq, seq = both(False)
        buf_par, par = both(True)
        where = f"rows {rows}, columns [0, {n1}) and [{n1}, {n1 + n2}), lda {lda}"
        assert torch.equal(buf_par.isnan(), buf_seq.isnan()), f"lda padding or row pattern differs; {where}"
        assert torch.equal(seq, seq0), f"two sequential runs differ; {where}"
        assert torch.equal(par, seq), f"concurrent updates differ from sequential ones; {where}"
        assert torch.isnan(buf_seq.view(n1 + n2, lda)[:, rows:]).all(), f"lda padding written; {where}"
        assert torch.equal(seq[:5], a.C0[:5]), f"rows above row_lo changed; {where}"
        err1 = float((seq[5:, :n1] - a.Cexp[5:, :n1]).abs().max() / a.Cexp[5:, :n1].abs().max())
        err2 = float((seq[5:, n1:] - b.Cexp[5:, n1:]).abs().max() / b.Cexp[5:, n1:].abs().max())
        assert max(err1, err2) < 1e-13, f"relative errors {err1:.2e}, {err2:.2e}; {where}"
    finally:
        torch.cuda.synchronize()
        h1.close()
        h2.close()
