"""Option gemm_trace: clock64 buckets of the MMA warps of k_gemm_vta and k_gemm_cvy_p, one row per CTA of every traced launch
(include/dhqr.h).  The trace must not change a bit of the factorisation, every CTA of a traced launch must write its row, and
the buckets of a row, disjoint spans of its warps' lifetimes, must add up to no more than the lifetime word."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

M, N = 8192, 1024     # four panel pairs: k_gemm_vta<128>, and k_gemm_cvy_p at K = 256 (pair updates) and K = 128 (inner applies)
WORDS = 8


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def factor(D, h):
    dev = torch.device("cuda:0")
    A = D.colmajor_empty(M, N, dev)
    D.fill_uniform_(A, 3)
    al = torch.zeros(N, dtype=torch.float64, device=dev)
    D.householder_(A, al, 0, handle=h)
    torch.cuda.synchronize()
    return A.cpu().numpy(), al.cpu().numpy()


def rows_of(D, h):
    buf = torch.zeros(2 + WORDS * (1 << 17), dtype=torch.float64, device="cuda:0")
    D._lib.call("dhqr_debug_copy_f64", h.raw, b"gemm_trace", C.c_void_p(buf.data_ptr()), buf.numel(), None)
    b = buf.cpu().numpy()
    return b[2:2 + WORDS * int(b[0])].reshape(-1, WORDS), int(b[1])


def test_trace_changes_no_bit_and_every_cta_reports(D):
    h = D.Handle(0)
    try:
        H0, a0 = factor(D, h)
        h.set_option("gemm_trace", 1)
        H1, a1 = factor(D, h)
        h.set_option("gemm_trace", 0)
        rows, dropped = rows_of(D, h)
        H2, a2 = factor(D, h)                      # off again: nothing more is written
        rows_after, _ = rows_of(D, h)
    finally:
        h.close()
    assert np.array_equal(H0.view(np.uint64), H1.view(np.uint64)) and np.array_equal(a0.view(np.uint64), a1.view(np.uint64))
    assert np.array_equal(H0.view(np.uint64), H2.view(np.uint64)) and np.array_equal(a0.view(np.uint64), a2.view(np.uint64))
    assert dropped == 0 and len(rows) > 0
    assert np.array_equal(rows, rows_after)

    kinds = rows[:, 0].astype(np.int64)
    assert {(1 << 16) | 128, (2 << 16) | 128, (2 << 16) | 256} <= set(kinds) and set(kinds >> 16) == {1, 2}, sorted(set(kinds))
    life = rows[:, 7]
    assert (life > 0).all(), f"{int((life <= 0).sum())} of {len(rows)} rows never written"
    assert (rows[:, 1:7] >= 0).all()
    assert (rows[:, 1:7].sum(axis=1) <= life).all()
    cvy = kinds >> 16 == 2
    assert (rows[cvy, 3] > 0).all() and (rows[cvy, 5] > 0).all()   # every cvy CTA here has a real tile: k-loop and epilogue
    assert (rows[~cvy, 3] > 0).all()
