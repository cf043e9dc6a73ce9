"""The argument contract of every numerical entry point of include/dhqr.h, driven from one list.

For each of the 40 entry points: a valid argument list over one NaN-filled device buffer (and NaN-filled host arrays for the host
entries), and a table of single bad arguments with the code each returns.  Every rejected call must return its code without
enqueuing a launch and leave every byte of every buffer as it was; the calls whose check is inactive (an empty operand left null or
overlapping, k = 0, rank = 0, nrhs = 0) must return 0 and do the same.  Small shapes only, and a Float64 pointer that is not 8 B
aligned is passed only to the entry points that check it (the pivoted QR, the complete orthogonal decomposition, the append and
downdate and the batched ones)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SLOT = 4096                      # doubles per operand slot, far more than any operand below needs
m, n, r, k, bt, rk = 8, 4, 2, 3, 3, 2
BIG_K = 10 ** 7                  # above the rows one append or downdate can take on any device


@pytest.fixture(scope="module")
def D():
    assert torch.cuda.is_available()
    import dhqr_b200
    return dhqr_b200


@pytest.fixture(scope="module")
def h(D):
    hd = D.Handle(0)
    yield hd
    torch.cuda.synchronize()
    hd.close()


@pytest.fixture(scope="module")
def bufs():
    dev = torch.full((64 + 16 * SLOT,), float("nan"), dtype=torch.float64, device=DEV)
    host = {name: np.full(SLOT, np.nan) for name in ("A", "alpha", "b", "x")}
    torch.cuda.synchronize()
    return dev, host


def table(h, bufs):
    """entry point -> (valid arguments, {code: [(argument index, bad value)]}, [[(index, value), ...] that must return 0])"""
    dev, host = bufs
    base = dev.data_ptr() + 8 * 64
    slot = {s: base + 8 * SLOT * i for i, s in enumerate(("A", "al", "b", "Q", "jp", "F", "g", "R", "B", "vt", "c", "e", "info", "out"))}
    P = {s: C.c_void_p(p) for s, p in slot.items()}
    mis = {s: C.c_void_p(p + 4) for s, p in slot.items()}          # not 8 B aligned (only where Float64 alignment is checked)
    cmis = {s: C.c_void_p(p + 8) for s, p in slot.items()}         # 8 B but not 16 B aligned (ComplexF64)
    over = {s: C.c_void_p(p + 16) for s, p in slot.items()}        # inside the operand of that slot, aligned for either type
    H = {s: C.c_void_p(a.ctypes.data) for s, a in host.items()}
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    hd, A, al, b, Q, jp, F, g, R, B, vt, c, e, info, out = (h.raw, *(P[s] for s in ("A", "al", "b", "Q", "jp", "F", "g", "R", "B", "vt",
                                                                                    "c", "e", "info", "out")))
    T = {}

    # ---- the column-block entry points: handle, m, n_global, col0, n_local, A, lda, ... --------------------------------------
    blk = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, m + 1)], -4: [(3, -1), (3, n + 1)], -5: [(4, -1), (4, n + 1), (3, 1)],
           -6: [(5, None)], -7: [(6, m - 1), (6, 0)]}
    empty = [[(2, 0), (4, 0), (5, None)]]                          # n_global = n_local = 0 with a null A
    T["dhqr_qr_f64"] = ([hd, m, n, 0, n, A, m, al, 0, st], {**blk, -8: [(7, None)], -9: [(8, 2), (8, 48), (8, 160), (8, -32)]},
                        [[(2, 0), (4, 0), (5, None), (7, None)]])
    for fn in ("dhqr_apply_qt_f64", "dhqr_apply_q_f64"):
        T[fn] = ([hd, m, n, 0, n, A, m, b, m, r, st], {**blk, -8: [(7, None)], -9: [(8, m - 1)], -10: [(9, -1)]},
                 empty + [[(7, None), (9, 0)]])
    T["dhqr_backsolve_f64"] = ([hd, m, n, 0, n, A, m, al, b, m, r, st],
                               {**blk, -8: [(7, None)], -9: [(8, None)], -10: [(9, m - 1)], -11: [(10, -1)]},
                               [[(2, 0), (4, 0), (5, None), (7, None)], [(8, None), (10, 0)]])
    # b, ldb and nrhs of dhqr_solve_f64 return the codes of their places in dhqr_apply_qt_f64
    T["dhqr_solve_f64"] = ([hd, m, n, 0, n, A, m, al, b, m, r, st],
                           {**blk, -8: [(7, None), (8, None)], -9: [(9, m - 1)], -10: [(10, -1)]},
                           [[(2, 0), (4, 0), (5, None), (7, None)], [(8, None), (10, 0)]])
    cblk = {**blk, -1: blk[-1] + [(4, n - 1)], -6: blk[-6] + [(5, cmis["A"])]}
    T["dhqr_qr_c64"] = ([hd, m, n, 0, n, A, m, al, st], {**cblk, -8: [(7, None), (7, cmis["al"])]},
                        [[(2, 0), (4, 0), (5, None), (7, None)]])
    T["dhqr_apply_qt_c64"] = ([hd, m, n, 0, n, A, m, b, m, r, st],
                              {**cblk, -8: [(7, None), (7, cmis["b"])], -9: [(8, m - 1)], -10: [(9, -1)]}, empty + [[(7, None), (9, 0)]])
    for fn in ("dhqr_backsolve_c64", "dhqr_solve_c64"):
        T[fn] = ([hd, m, n, 0, n, A, m, al, b, m, r, st],
                 {**cblk, -8: [(7, None), (7, cmis["al"])], -9: [(8, None), (8, cmis["b"])], -10: [(9, m - 1)], -11: [(10, -1)]},
                 [[(2, 0), (4, 0), (5, None), (7, None)], [(8, None), (10, 0)]])

    # ---- host entries: hA, lda and h_alpha return the codes of dA_local, lda and d_alpha of dhqr_qr_f64 ----------------------
    hosthead = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, m + 1)], -6: [(3, None), (5, None)], -7: [(4, m - 1)]}
    T["dhqr_qr_host_f64"] = ([hd, m, n, H["A"], m, H["alpha"], 0], {**hosthead, -9: [(6, 2), (6, 100)]},
                             [[(2, 0), (3, None), (5, None)]])
    T["dhqr_ldiv_host_f64"] = ([hd, m, n, H["A"], m, H["alpha"], H["b"], H["x"]], {**hosthead, -7: [(4, m - 1), (6, None)], -8: [(7, None)]},
                               [[(2, 0), (3, None), (5, None), (7, None)]])

    # ---- primitives ----------------------------------------------------------------------------------------------------------
    pd = {-1: [(0, None)], -2: [(1, None)], -3: [(2, None)], -4: [(3, -1)], -5: [(4, -1)], -6: [(5, None)]}
    T["dhqr_partialdot_f64"] = ([hd, A, b, 0, m, out, st], pd, [])
    T["dhqr_partialdot_c64"] = ([hd, A, b, 0, m, out, st], {**pd, -2: [(1, None), (1, cmis["A"])], -3: [(2, None), (2, cmis["b"])],
                                                            -6: [(5, None), (5, cmis["out"])]}, [])
    T["dhqr_fill_uniform_f64"] = ([hd, 1, 0, 0, m, n, A, m, st], {-1: [(0, None)], -5: [(4, -1)], -6: [(5, -1)], -7: [(6, None)],
                                                                   -8: [(7, m - 1)]}, [[(4, 0), (6, None)], [(5, 0), (6, None)]])

    # ---- single-GPU entry points: handle, m, n, ... --------------------------------------------------------------------------
    mn = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, m + 1)]}
    for t, bad in (("f64", lambda s: []), ("c64", lambda s: [cmis[s]])):
        T[f"dhqr_form_q_{t}"] = ([hd, m, n, A, m, Q, m, st],
                                 {**mn, -4: [(3, v) for v in [None] + bad("A")], -5: [(4, m - 1)],
                                  -6: [(5, v) for v in [None, over["A"]] + bad("Q")], -7: [(6, m - 1)]},
                                 [[(2, 0), (3, None), (5, None)], [(2, 0), (5, A)]])
        for fn in (f"dhqr_forwardsolve_{t}", f"dhqr_solve_adj_{t}"):
            T[fn] = ([hd, m, n, A, m, al, b, m, r, st],
                     {**mn, -4: [(3, v) for v in [None] + bad("A")], -5: [(4, m - 1)], -6: [(5, v) for v in [None] + bad("al")],
                      -7: [(6, v) for v in [None] + bad("b")], -8: [(7, m - 1)], -9: [(8, -1)]},
                     [[(6, None), (8, 0)]] + ([[(2, 0), (3, None), (5, None)]] if fn.startswith("dhqr_forward") else []))
    for t, mz in (("f64", mis), ("c64", cmis)):
        T[f"dhqr_qrcp_{t}"] = ([hd, m, n, A, m, al, jp, st],
                               {**mn, -4: [(3, None), (3, mz["A"])], -5: [(4, m - 1)], -6: [(5, None), (5, mz["al"])],
                                -7: [(6, None), (6, mis["jp"])]}, [[(2, 0), (3, None), (5, None), (6, None)]])
        rnk = {**mn, -4: [(3, -1), (3, n + 1)], -5: [(4, None), (4, mz["A"])], -6: [(5, m - 1)]}
        T[f"dhqr_solve_qrcp_{t}"] = ([hd, m, n, rk, A, m, al, jp, b, m, r, st],
                                     {**rnk, -7: [(6, None), (6, mz["al"])], -8: [(7, None), (7, mis["jp"])],
                                      -9: [(8, None), (8, mz["b"])], -10: [(9, m - 1)], -11: [(10, -1)]}, [[(8, None), (10, 0)]])
        T[f"dhqr_cod_{t}"] = ([hd, m, n, rk, A, m, al, F, n, g, st],
                              {**rnk, -7: [(6, None), (6, mz["al"])], -8: [(7, None), (7, mz["F"]), (7, A), (7, al)], -9: [(8, n - 1)],
                               -10: [(9, None), (9, mz["g"]), (9, A), (9, al), (9, F)]},
                              [[(3, 0), (7, None), (9, None)], [(3, 0), (7, A), (9, al)]])
        T[f"dhqr_solve_cod_{t}"] = ([hd, m, n, rk, A, m, jp, F, n, g, b, m, r, st],
                                    {**rnk, -7: [(6, None), (6, mis["jp"])], -8: [(7, None), (7, mz["F"])], -9: [(8, n - 1)],
                                     -10: [(9, None), (9, mz["g"])], -11: [(10, None), (10, mz["b"])], -12: [(11, m - 1)], -13: [(12, -1)]},
                                    [[(10, None), (12, 0)], [(7, A), (9, al), (10, None), (12, 0)]])

    # ---- append and downdate: handle, n, k, ... ------------------------------------------------------------------------------
    nk = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (2, BIG_K)]}
    tp = {**nk, -4: [(3, None), (3, mis["R"])], -5: [(4, n - 1)], -6: [(5, None), (5, mis["al"])],
          -7: [(6, None), (6, mis["B"]), (6, R), (6, al)], -8: [(7, k - 1)], -9: [(8, None), (8, mis["vt"]), (8, R), (8, al), (8, B)]}
    tp0 = [[(2, 0), (6, None)], [(2, 0), (8, R)]]                  # k = 0: B may be null, vtop may overlap
    T["dhqr_qr_append_f64"] = ([hd, n, k, R, n, al, B, k, vt, st], tp, tp0)
    T["dhqr_qr_downdate_f64"] = ([hd, n, k, R, n, al, B, k, vt, info, st],
                                 {**tp, -10: [(9, None), (9, mis["info"]), (9, R), (9, al), (9, B), (9, vt)]},
                                 [tp0[0] + [(9, None)], tp0[1]])
    for fn in ("dhqr_apply_qt_append_f64", "dhqr_apply_q_append_f64", "dhqr_apply_downdate_f64"):
        T[fn] = ([hd, n, k, B, k, vt, c, n, e, k, r, st],
                 {**nk, -4: [(3, None), (3, mis["B"])], -5: [(4, k - 1)], -6: [(5, None), (5, mis["vt"])],
                  -7: [(6, None), (6, mis["c"]), (6, B), (6, vt)], -8: [(7, n - 1)],
                  -9: [(8, None), (8, mis["e"]), (8, B), (8, vt), (8, c)], -10: [(9, k - 1)], -11: [(10, -1)]},
                 [[(6, None), (8, None), (10, 0)], [(2, 0), (3, None), (8, None)]])

    # ---- batched: handle, m, n, batch, A, lda, stride_a, ... -----------------------------------------------------------------
    bh = {**mn, -3: mn[-3] + [(1, 60000)], -4: [(3, -1), (3, 2 ** 31)], -5: [(4, None), (4, mis["A"])], -6: [(5, m - 1)],
          -7: [(6, m * n - 1)]}                                     # m = 60000: m * n above batch_max_elems
    T["dhqr_qr_batched_f64"] = ([hd, m, n, bt, A, m, m * n, al, n, st],
                                {**bh, -8: [(7, None), (7, mis["al"]), (7, A)], -9: [(8, n - 1)]}, [[(3, 0), (4, None), (7, None)]])
    for fn in ("dhqr_apply_qt_batched_f64", "dhqr_apply_q_batched_f64"):
        T[fn] = ([hd, m, n, bt, A, m, m * n, b, m, m * r, r, st],
                 {**bh, -8: [(7, None), (7, mis["b"]), (7, A)], -9: [(8, m - 1)], -10: [(9, m * r - 1)], -11: [(10, -1)]},
                 [[(7, None), (10, 0)], [(3, 0), (4, None), (7, None)]])
    T["dhqr_solve_batched_f64"] = ([hd, m, n, bt, A, m, m * n, al, n, b, m, m * r, r, st],
                                   {**bh, -8: [(7, None), (7, mis["al"]), (7, A)], -9: [(8, n - 1)], -10: [(9, None), (9, mis["b"]), (9, A), (9, al)],
                                    -11: [(10, m - 1)], -12: [(11, m * r - 1)], -13: [(12, -1)]},
                                   [[(9, None), (12, 0)], [(3, 0), (4, None), (7, None), (9, None)]])
    up = {-1: [(0, None)], -2: [(1, -1)], -3: [(2, -1), (1, 1025)], -4: [(3, -1)], -5: [(4, None), (4, mis["R"])], -6: [(5, n - 1)],
          -7: [(6, n * n - 1)], -8: [(7, None), (7, mis["al"]), (7, R)], -9: [(8, n - 1)], -10: [(9, None), (9, mis["B"]), (9, R), (9, al)],
          -11: [(10, k - 1)], -12: [(11, k * n - 1)], -13: [(12, None), (12, mis["vt"]), (12, R), (12, al), (12, B)], -14: [(13, n - 1)],
          -15: [(14, None), (14, mis["c"]), (14, R), (14, al), (14, B), (14, vt)], -16: [(15, n - 1)], -17: [(16, n * r - 1)],
          -18: [(17, None), (17, mis["e"]), (17, R), (17, al), (17, B), (17, vt), (17, c)], -19: [(18, k - 1)], -20: [(19, k * r - 1)],
          -21: [(20, -1)]}
    ap = [hd, n, k, bt, R, n, n * n, al, n, B, k, k * n, vt, n, c, n, n * r, e, k, k * r, r, st]
    up0 = [[(3, 0), (4, None), (7, None), (9, None), (12, None), (14, None), (17, None)],
           [(2, 0), (9, None), (12, R), (14, R), (17, R)]]          # batch = 0; k = 0: nothing is written, so nothing may overlap
    T["dhqr_qr_append_batched_f64"] = (ap, up, up0)
    T["dhqr_qr_downdate_batched_f64"] = (ap[:-1] + [info, st],
                                         {**up, -22: [(21, None), (21, mis["info"]), (21, R), (21, al), (21, B), (21, vt), (21, c), (21, e)]},
                                         [up0[0] + [(21, None)], up0[1] + [(21, R)]])
    T["dhqr_backsolve_batched_f64"] = ([hd, n, bt, R, n, n * n, al, n, c, n, n * r, r, st],
                                       {-1: [(0, None)], -2: [(1, -1), (1, 1025)], -3: [(2, -1), (2, 2 ** 31)], -4: [(3, None), (3, mis["R"])],
                                        -5: [(4, n - 1)], -6: [(5, n * n - 1)], -7: [(6, None), (6, mis["al"])], -8: [(7, n - 1)],
                                        -9: [(8, None), (8, mis["c"]), (8, R), (8, al)], -10: [(9, n - 1)], -11: [(10, n * r - 1)],
                                        -12: [(11, -1)]},
                                       [[(8, None), (11, 0)], [(2, 0), (3, None), (6, None)], [(6, R), (8, None), (11, 0)]])
    return T


NAMES = ["dhqr_qr_f64", "dhqr_apply_qt_f64", "dhqr_apply_q_f64", "dhqr_backsolve_f64", "dhqr_solve_f64", "dhqr_qr_c64",
         "dhqr_apply_qt_c64", "dhqr_backsolve_c64", "dhqr_solve_c64", "dhqr_qr_host_f64", "dhqr_ldiv_host_f64", "dhqr_partialdot_f64",
         "dhqr_partialdot_c64", "dhqr_fill_uniform_f64", "dhqr_form_q_f64", "dhqr_form_q_c64", "dhqr_forwardsolve_f64",
         "dhqr_forwardsolve_c64", "dhqr_solve_adj_f64", "dhqr_solve_adj_c64", "dhqr_qrcp_f64", "dhqr_qrcp_c64", "dhqr_solve_qrcp_f64",
         "dhqr_solve_qrcp_c64", "dhqr_cod_f64", "dhqr_cod_c64", "dhqr_solve_cod_f64", "dhqr_solve_cod_c64", "dhqr_qr_append_f64",
         "dhqr_qr_downdate_f64", "dhqr_apply_qt_append_f64", "dhqr_apply_q_append_f64", "dhqr_apply_downdate_f64",
         "dhqr_qr_batched_f64", "dhqr_apply_qt_batched_f64", "dhqr_apply_q_batched_f64", "dhqr_solve_batched_f64",
         "dhqr_qr_append_batched_f64", "dhqr_qr_downdate_batched_f64", "dhqr_backsolve_batched_f64"]


def test_the_list_is_every_numerical_entry_point(D, h, bufs):
    assert len(NAMES) == 40 and sorted(NAMES) == sorted(table(h, bufs))


def _snapshot(bufs):
    dev, host = bufs
    torch.cuda.synchronize()
    return dev.view(torch.int64).clone(), {s: a.view(np.int64).copy() for s, a in host.items()}


def _unchanged(bufs, snap):
    dev, host = bufs
    torch.cuda.synchronize()
    return torch.equal(dev.view(torch.int64), snap[0]) and all(np.array_equal(a.view(np.int64), snap[1][s]) for s, a in host.items())


def _call(D, fn, args, subs):
    a = list(args)
    for idx, val in subs:
        a[idx] = val
    return getattr(D._lib.load(), fn)(*a)


@pytest.mark.parametrize("fn", NAMES)
def test_rejected_call_changes_nothing(D, h, bufs, fn):
    """Each single bad argument returns its code, enqueues nothing and leaves every buffer bitwise as it was."""
    args, cases, _ = table(h, bufs)[fn]
    snap = _snapshot(bufs)
    for code, subs in cases.items():
        for idx, val in subs:
            l0 = h.launch_count()
            rc = _call(D, fn, args, [(idx, val)])
            assert rc == code, (fn, idx, val, rc, code, D._lib.load().dhqr_last_error())
            assert h.launch_count() == l0, (fn, idx, val, "launched")
            assert _unchanged(bufs, snap), (fn, idx, val, "wrote")


@pytest.mark.parametrize("fn", [f for f in NAMES if f not in ("dhqr_partialdot_f64", "dhqr_partialdot_c64")])
def test_inactive_checks_return_0(D, h, bufs, fn):
    """An empty operand may be null or overlap another one: the call returns 0 and, having nothing to do, does nothing."""
    args, _, empties = table(h, bufs)[fn]
    assert empties
    snap = _snapshot(bufs)
    for subs in empties:
        l0 = h.launch_count()
        rc = _call(D, fn, args, subs)
        assert rc == 0, (fn, subs, rc, D._lib.load().dhqr_last_error())
        assert h.launch_count() == l0 and _unchanged(bufs, snap), (fn, subs)
