"""The first two stages of the 128-column panel chain after the pack was folded into the first Gram pass (k_pack_gram) and
the second Gram matrix into the first solve pass (k_vpk_rmul in Gram mode): G1 (through R1 = chol(G1)), G2 = Q1'Q1 (the
reduced sum left in wsum) and the packed V block, against torch fp64 products, for aligned storage, an odd leading
dimension, a base 8 bytes off 16 B alignment and ragged windows.  Bulk-copy and generic staging of the panel's columns must
agree bitwise, and so must two runs."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROWS = [128, 129, 200, 1000, 4097, 8192]
LAYOUTS = ["aligned", "odd_lda", "offset8"]


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def vp(t):
    return C.c_void_p(t.data_ptr())


def sp():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def debug_copy(D, what, n):
    buf = torch.zeros(n, dtype=torch.float64, device="cuda:0")
    D._lib.call("dhqr_debug_copy_f64", D.default_handle(0).raw, what, vp(buf), n, sp())
    torch.cuda.synchronize()
    return buf


def run_panel(D, P, layout):
    """Factor the panel P (rows x 128) stored as `layout`; returns H, alpha, R1, G2 and the packed V, all as numpy."""
    rows = P.shape[0]
    lda = rows + (rows % 2) if layout != "odd_lda" else rows + 1 - (rows % 2)
    off = 1 if layout == "offset8" else 0
    store = torch.zeros(lda * 128 + 2, dtype=torch.float64, device="cuda:0")
    dP = torch.as_strided(store, (rows, 128), (1, lda), off)
    dP.copy_(torch.from_numpy(P))
    assert (dP.data_ptr() % 16 == 0) == (layout != "offset8") and (lda % 2 == 1) == (layout == "odd_lda")
    dal = torch.zeros(128, dtype=torch.float64, device="cuda:0")
    refused = C.c_int(-1)
    D._lib.call("dhqr_k_wide_panel_f64", D.default_handle(0).raw, rows, vp(dP), lda, vp(dal), C.byref(refused), sp())
    torch.cuda.synchronize()
    assert refused.value == 0
    R1 = debug_copy(D, b"wide", 128 * 128).cpu().numpy().reshape(128, 128).T.copy()
    G2 = debug_copy(D, b"wsum", 128 * 128).cpu().numpy().reshape(128, 128).T.copy()
    vrows = (rows + 127) // 128 * 128
    V = debug_copy(D, b"vpk", vrows // 64 * 128 * 68).cpu().numpy().reshape(vrows // 64, 128, 68)
    return dP.cpu().numpy(), dal.cpu().numpy(), R1, G2, V


@pytest.mark.parametrize("rows", ROWS)
def test_gram_stages_against_torch(D, oracle, rows):
    P = oracle.np_uniform(40 + rows % 7, rows, 128)
    ref = None
    for layout in LAYOUTS:
        H, al, R1, G2, V = run_panel(D, P, layout)
        out = (H, al, R1, G2, V)
        if ref is None:
            ref = out
            tP = torch.from_numpy(P)
            G1 = (tP.T @ tP).numpy()
            tR1 = torch.from_numpy(R1)
            assert np.abs(np.tril(R1, -1)).max() == 0.0
            assert np.abs((tR1.T @ tR1).numpy() - G1).max() < 1e-13 * np.abs(G1).max(), "G1 (k_pack_gram) / k_chol128"
            Q1 = torch.linalg.solve_triangular(tR1, tP, upper=True, left=False)
            assert np.abs(G2 - (Q1.T @ Q1).numpy()).max() < 1e-12, "G2 (k_vpk_rmul in Gram mode)"
            assert np.abs(G2 - np.eye(128)).max() < 1e-9
            # the packed V block: tril(H) in rows 0..63 of every column, zero past the window
            Vd = V[:, :, :64].transpose(0, 2, 1).reshape(-1, 128)
            assert np.array_equal(Vd[:rows], np.tril(H)) and not Vd[rows:].any()
            assert oracle.qr_residual(P, np.asfortranarray(H), al) < 1e-13
            again = run_panel(D, P, layout)
            for a, b in zip(out, again):
                assert np.array_equal(a, b), "two runs differ"
        else:
            for name, a, b in zip(("H", "alpha", "R1", "G2", "vpk"), out, ref):
                if name == "vpk":
                    a, b = a[:, :, :64], b[:, :, :64]
                assert np.array_equal(a, b), f"{layout} differs from aligned storage in {name}"
