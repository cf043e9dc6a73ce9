"""The pipelined host entry (DESIGN 2.5) on the CPU: the PRODUCT's upload planner (dhqr_plan_host_upload, pure host logic in
libdhqr.so) is checked for the invariants the look-ahead driver relies on, and a numpy restatement of the windowed schedule —
window of arrived columns, catch-up of a late chunk with the reflectors already finished, join — driven by that plan must give the
reference factorisation (S:122-148, S:198-213): every column receives every reflector exactly once and in order."""
import numpy as np
import pytest

import dhqr_b200 as D


def windowed_qr(a, nb, bounds, join):
    """Right-looking QR in panels of nb columns on a window that grows by the plan: columns [wend, n) are 'not uploaded yet'.
    Returns (H, alpha, log) with log[c] = list of reflector indices applied to column c, in order."""
    from dhqr_oracle import np_alphafactor
    h = np.array(a, dtype=np.float64, order="F", copy=True)
    m, n = h.shape
    alpha = np.zeros(n)
    K = (n + nb - 1) // nb
    log = [[] for _ in range(n)]
    wend = bounds[1]
    nxt = 1

    def apply_panel(q, c0, c1):                            # reflectors of panel q -> columns [c0, c1)
        for j in range(q * nb, min(n, (q + 1) * nb)):
            v = h[j:, j]
            if c1 > c0:
                s = v @ h[j:, c0:c1]                       # S:208
                h[j:, c0:c1] -= np.outer(v, s)             # S:209
                for c in range(c0, c1):
                    log[c].append(j)

    for k in range(K):
        p0, p1 = k * nb, min(n, (k + 1) * nb)
        t2 = min(n, (k + 3) * nb)                          # end of panel k+2
        t3 = min(n, (k + 4) * nb)                          # end of panel k+3
        joined = []
        while nxt < len(bounds) - 1 and (join[nxt] <= k or bounds[nxt] < t3):     # the driver's rule (qr_blocked_lookahead)
            assert bounds[nxt] >= t2 and bounds[nxt] == wend, "chunk joins too late"
            for q in range(k):                             # catch-up: panels 0 .. k-1, in order
                apply_panel(q, bounds[nxt], bounds[nxt + 1])
            joined.append((bounds[nxt], bounds[nxt + 1]))
            wend = bounds[nxt + 1]
            nxt += 1
        assert wend >= t2, "window ends before panel k+2"
        wold = joined[0][0] if joined else wend
        for j in range(p0, p1):                            # the panel itself, column by column (S:127-135, S:208-209 inside the panel)
            assert p1 <= wold
            s = np.linalg.norm(h[j:, j])
            alpha[j] = s * np_alphafactor(h[j, j])
            f = 1.0 / np.sqrt(s * (s + abs(h[j, j])))
            h[j, j] -= alpha[j]
            h[j:, j] *= f
            v = h[j:, j]
            if j + 1 < p1:
                sa = v @ h[j:, j + 1:p1]
                h[j:, j + 1:p1] -= np.outer(v, sa)
                for c in range(j + 1, p1):
                    log[c].append(j)
        apply_panel(k, p1, wold)                           # chain / hp2 / bulk: everything right of the panel inside the old window
        for c0, c1 in joined:                              # the chunks that joined at this step, behind their catch-up
            apply_panel(k, c0, c1)
    assert nxt == len(bounds) - 1 and wend == n
    return h, alpha, log


CASES = [(32768, 4096, 128), (65536, 8192, 128), (4096, 2176, 128), (3000, 1408, 128), (2304, 1152, 96), (2304, 1152, 64), (2304, 1152, 32),
         (5000, 5000, 128), (1024, 128, 128), (2500, 1100, 128)]
MODELS = [dict(), dict(chunk=128, h2d_gbs=1), dict(chunk=128, h2d_gbs=100000), dict(chunk=256), dict(chunk=384, h2d_gbs=3),
          dict(chunk=1024, chain_us=2500), dict(chunk=512, first=768, chain_us=1000), dict(chunk=0)]


@pytest.mark.parametrize("mnb", CASES)
def test_plan_invariants(mnb):
    m, n, nb = mnb
    for kw in MODELS:
        b, j = D.plan_host_upload(m, n, nb, **kw)
        assert b[0] == 0 and b[-1] == n and len(j) == len(b) - 1 and j[0] == 0
        assert all(b[i] < b[i + 1] for i in range(len(b) - 1))
        assert all(x % nb == 0 for x in b[:-1])
        if len(b) > 2:
            assert b[1] >= 3 * nb                                       # the schedule starts on panels 0..2
            assert all(j[i] <= j[i + 1] for i in range(len(j) - 1))
            assert all(0 <= j[i] <= b[i] // nb - 3 for i in range(1, len(j))), (kw, b, j)   # never later than the deadline
        if kw.get("chunk", 512) == 0:
            assert b == [0, n]


def test_default_plan_of_the_bench_workload():
    b, j = D.plan_host_upload(32768, 4096)
    assert b == [0, 384, 768, 1280, 1792, 2304, 2816, 3328, 3840, 4096]
    assert j == [0, 0, 3, 7, 11, 15, 19, 23, 27]                       # deadline joins


@pytest.mark.parametrize("mnb", [(700, 640, 32), (900, 768, 64), (1300, 1152, 96), (1100, 1024, 128)])
def test_windowed_schedule_gives_the_reference_factorisation(oracle, mnb):
    m, n, nb = mnb
    A = oracle.np_uniform(21, m, n)
    Href, aref = oracle.np_qr(A)
    for kw in (dict(chunk=nb), dict(chunk=nb, h2d_gbs=100000), dict(chunk=2 * nb, chain_us=2000), dict(chunk=nb, h2d_gbs=1, first=5 * nb)):
        b, j = D.plan_host_upload(m, n, nb, **kw)
        assert len(b) > 2, "the case must exercise the pipeline"
        H, a, log = windowed_qr(A, nb, b, j)
        for c in range(n):
            assert log[c] == list(range(c)), (kw, c)                    # every reflector left of the column, once, in order
        assert np.abs(H - Href).max() < 1e-12 and np.abs(a - aref).max() < 1e-12 * np.abs(aref).max()


def test_bad_arguments():
    lib = D._lib.load()
    import ctypes as C
    b, j, k = (C.c_int64 * 8)(), (C.c_int * 8)(), C.c_int()
    assert lib.dhqr_plan_host_upload(10, 20, 128, 512, 0, 50, 27, 300, 8, b, j, C.byref(k)) == -2       # n > m
    assert lib.dhqr_plan_host_upload(4096, 4096, 100, 512, 0, 50, 27, 300, 8, b, j, C.byref(k)) == -3   # nb
    assert lib.dhqr_plan_host_upload(32768, 4096, 128, 512, 0, 50, 27, 300, 4, b, j, C.byref(k)) == -9  # cap
    assert lib.dhqr_plan_host_upload(32768, 4096, 128, 512, 0, 50, 27, 300, 8, None, j, C.byref(k)) == -10


def driver_accepts(n, nb, bounds, join):
    """The join rule of qr_blocked_lookahead without the numerics: True when every chunk joins while it still lies right of
    panel k+2 and the window always reaches panel k+2 (the driver's internal errors 4005 can then not occur)."""
    K = (n + nb - 1) // nb
    wend, nxt = bounds[1], 1
    for k in range(K):
        t2, t3 = min(n, (k + 3) * nb), min(n, (k + 4) * nb)
        while nxt < len(bounds) - 1 and (join[nxt] <= k or bounds[nxt] < t3):
            if bounds[nxt] < t2 or bounds[nxt] != wend:
                return False
            wend = bounds[nxt + 1]
            nxt += 1
        if wend < t2:
            return False
    return nxt == len(bounds) - 1 and wend == n


def test_no_option_setting_can_trip_the_driver():
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=400, deadline=None)
    @given(nb=st.sampled_from([32, 64, 96, 128]), npan=st.integers(1, 80), ragged=st.integers(0, 127), extra=st.integers(0, 5000),
           chunk=st.integers(0, 12), first=st.integers(0, 3000), gbs=st.integers(1, 2000), tf=st.integers(1, 200),
           chain=st.integers(1, 20000))
    def check(nb, npan, ragged, extra, chunk, first, gbs, tf, chain):
        n = max(1, npan * nb - (ragged % nb))
        m = n + extra
        b, j = D.plan_host_upload(m, n, nb, chunk=128 * chunk, first=first, h2d_gbs=gbs, tflops=tf, chain_us=chain)
        assert b[0] == 0 and b[-1] == n and len(j) == len(b) - 1
        assert driver_accepts(n, nb, b, j), (m, n, nb, b, j)

    check()
