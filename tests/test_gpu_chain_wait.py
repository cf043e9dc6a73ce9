"""Option chain_wait_trace: every launch on the look-ahead schedule's chain streams gets CUDA events around it and %globaltimer
stamps from its kernel (first CTA start, last warp end).  The trace must leave the factorisation bitwise unchanged, and stamp
every launch it records, with the stamp span inside the event span up to the clocks' resolution."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def factor(D, h, m, n):
    A = D.colmajor_empty(m, n, "cuda:0")
    D.fill_uniform_(A, 5, handle=h)
    al = torch.zeros(n, dtype=torch.float64, device="cuda:0")
    D.householder_(A, al, 0, handle=h)
    torch.cuda.synchronize()
    return A.cpu().numpy(), al.cpu().numpy()


def test_trace_stamps_every_chain_launch_and_changes_nothing(D):
    h = D.Handle(0)
    try:
        m, n = 8192, 1024                       # 8 wide panels: 4 pair units under the look-ahead schedule
        A0, a0 = factor(D, h, m, n)
        h.set_option("chain_wait_trace", 1)
        A1, a1 = factor(D, h, m, n)
        h.set_option("chain_wait_trace", 0)
        assert np.array_equal(A0, A1) and np.array_equal(a0, a1)

        buf = torch.zeros(1 + 6 * 8192, dtype=torch.float64, device="cuda:0")
        D._lib.call("dhqr_debug_copy_f64", h.raw, b"chain_wait", C.c_void_p(buf.data_ptr()), buf.numel(), None)
        b = buf.cpu().numpy()
        rows = b[1:1 + 6 * int(b[0])].reshape(-1, 6)
        assert len(rows) > 0
        unit, stream, cls, span, run, wait = rows.T
        assert set(stream.astype(int)) <= {0, 1, 2} and 0 in set(stream.astype(int))
        assert unit.min() == 0 and unit.max() <= 4
        assert (run >= 0).all(), "a chain launch without stamps"
        assert np.allclose(wait, span - run)
        assert (wait > -0.01).all()             # event timestamps are kept to about half a microsecond
        names = set()
        for c in sorted(set(cls.astype(int))):
            s = C.create_string_buffer(64)
            D._lib.call("dhqr_profile_get", h.raw, c, s, 64, None, None, None)
            names.add(s.value.decode())
        assert {"k_gram128", "k_chol128", "k_hr128", "k_gemm_cvy256"} <= names, names
    finally:
        h.close()
