"""The block-reflector update C <- (I - V T' V') C on rows >= row_lo (k_gemm_vta + k_wreduce + k_tinv + k_ymake + k_gemm_cvy_p)
at the edges of its 16x8x8 DMMA fragments and 128 x 64 tiles: row counts around 8, 16, 64 and 128, row_lo inside the first
fragment rows, column counts around 8 and 64, lda = rows and rows + 1 (odd leading dimensions take the generic-load fill
instead of the bulk copies).  Against torch fp64, with NaN in the lda padding rows, the rows above row_lo bitwise untouched,
two runs bitwise equal, and cvy_persist = 0 (one tile per CTA) bitwise equal to the default walk."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

ROWS = [1, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 4099]
ROW_LO = [0, 7, 8, 9, 16]
NCOLS = [1, 7, 8, 9, 63, 64, 65, 200]


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def householder_block(rows, row_lo, nbp, seed):
    """rows x nbp: reflectors with |v|^2 = 2 (or 0) on rows >= row_lo, zero above; columns past the last reflector are zero."""
    g = torch.Generator().manual_seed(seed)
    a, tau = torch.geqrf(torch.rand(rows - row_lo, nbp, dtype=torch.float64, generator=g))
    k = tau.numel()
    Vk = torch.tril(a[:, :k], -1) + torch.eye(rows - row_lo, k, dtype=torch.float64)
    V = torch.zeros(rows, nbp, dtype=torch.float64)
    V[row_lo:, :k] = Vk * tau.sqrt()
    return V


def apply(D, h, V, dV, C0, row_lo, lda):
    rows, ncols = C0.shape
    buf = torch.full((ncols * lda,), float("nan"), dtype=torch.float64, device=dV.device)
    dC = buf.as_strided((rows, ncols), (1, lda))
    dC.copy_(C0)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    D._lib.call("dhqr_k_block_reflector_f64", h.raw, rows, V.shape[1], C.c_void_p(dV.data_ptr()), rows, row_lo, ncols,
                C.c_void_p(buf.data_ptr()), lda, None, stream)
    torch.cuda.synchronize()
    return buf, dC


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("nbp", [128, 100])
def test_block_reflector_edges(D, nbp, rows):
    dev = torch.device("cuda:0")
    h = D.default_handle(0)
    persist = h.get_option("cvy_persist")
    try:
        for row_lo in [r for r in ROW_LO if r < rows]:
            V = householder_block(rows, row_lo, nbp, seed=rows * 131 + row_lo)
            dV = D.to_colmajor(V, dev)
            Vd = V.to(dev)
            L = torch.eye(nbp, dtype=torch.float64, device=dev) + torch.tril(Vd.T @ Vd, -1)
            Linv = torch.linalg.solve_triangular(L, torch.eye(nbp, dtype=torch.float64, device=dev), upper=False)
            for ncols in NCOLS:
                C0 = torch.rand(rows, ncols, dtype=torch.float64, device=dev,
                                generator=torch.Generator(device=dev).manual_seed(ncols))
                Cexp = C0 - Vd @ (Linv @ (Vd.T @ C0))
                for lda in (rows, rows + 1):
                    where = f"nbp {nbp}, rows {rows}, row_lo {row_lo}, ncols {ncols}, lda {lda}"
                    h.set_option("cvy_persist", persist)
                    buf, dC = apply(D, h, V, dV, C0, row_lo, lda)
                    if lda > rows:
                        assert torch.isnan(buf.view(ncols, lda)[:, rows:]).all(), f"lda padding written; {where}"
                    assert torch.equal(dC[:row_lo], C0[:row_lo]), f"rows above row_lo changed; {where}"
                    err = float((dC[row_lo:] - Cexp[row_lo:]).abs().max() / Cexp[row_lo:].abs().max())
                    assert err < 1e-13, f"relative error {err:.2e}; {where}"
                    _, dC2 = apply(D, h, V, dV, C0, row_lo, lda)
                    assert torch.equal(dC, dC2), f"two runs differ; {where}"
                    h.set_option("cvy_persist", 0)
                    _, dC3 = apply(D, h, V, dV, C0, row_lo, lda)
                    assert torch.equal(dC, dC3), f"cvy_persist = 0 differs from the default walk; {where}"
    finally:
        h.set_option("cvy_persist", persist)
