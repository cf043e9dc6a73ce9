"""When the library's work runs relative to the caller's (run with -m gpu on an H100).

include/dhqr.h promises that work is enqueued on the caller's stream, that nothing outside its four synchronisation points
blocks the host, and that no call depends on any stream but the caller's.  Inside, the schedule fans out over the handle's own
non-blocking streams (panel chain, second apply, wide-chain side kernels, collectives, host-entry copies) and is joined back to
the caller's stream by events.  A missing edge only shows when the caller's stream is busy or is read before a host sync, so
every case here runs behind a closed gate:

  1. warm-up: the case once, ungated, on the same handle (workspace growth, synchronisation point (iv), is not part of the
     gated call); reference: once more on the legacy stream, synchronised;
  2. gated: every buffer is filled with a decoy (another seeded matrix / right-hand side of the same shape and family, finite),
     the gate closes on stream S, and on S the true inputs are copied in, the call is made through the C-ABI, every output is
     copied to a snapshot and every buffer is overwritten with the decoy again: a side stream still reading after the call
     "returned" on S sees the decoy;
  3. the call must return with the gate still closed, unless dhqr.h lists it as a synchronisation point (a qr that ran a panel
     through the 128-column chain); after a synchronise the snapshots must be bitwise equal to the reference: same handle,
     same options and same inputs are the same arithmetic.

The gate is torch.cuda._sleep on a helper stream, an event recorded behind it, and S waiting on that event: one single-thread
CTA that ends by itself whatever the library does, so no outcome can leave anything waiting.  Between closing a gate and the
end of the calls the test does nothing that blocks the host (no .cpu(), .item() or fresh allocations).  The calibrated gate
length is written to build/test_gpu_streams_gate.txt.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import matrix_families as F
from ext_rule import COUNTERS, counters, options

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GATE_MS = 200.0          # long enough to cover the enqueue of the largest case here (a 2048 x 1024 factorisation and its copies)
FAMILY = "normal"        # every 128-column panel goes through the wide chain at 2048 x 1024 (test_gpu_shapes.py, ACCEPTED)
M2, N2 = 2048, 1024      # shape of the blocked cases and of the factorisation the solve cases read
MC, NC = 1000, 300       # ComplexF64 shape
MF, NF = 4096, 512       # fresh-handle shape: every first call of the sequence sizes the same workspace (no cudaFree in between)


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="module")
def h(D):
    hd = D.Handle(0)
    yield hd
    torch.cuda.synchronize()
    hd.close()


class Gate:
    """torch.cuda._sleep(cycles) on a helper stream; close(s) makes s wait for it and returns the event that opens it."""

    def __init__(self):
        self.g = torch.cuda.Stream()
        probe = 10_000_000
        rates = []
        for _ in range(4):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(self.g)
            with torch.cuda.stream(self.g):
                torch.cuda._sleep(probe)
            e1.record(self.g)
            e1.synchronize()
            rates.append(probe / e0.elapsed_time(e1))
        self.cycles_per_ms = float(np.median(rates[1:]))
        self.cycles = int(GATE_MS * self.cycles_per_ms)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.g)
        with torch.cuda.stream(self.g):
            torch.cuda._sleep(self.cycles)
        e1.record(self.g)
        e1.synchronize()
        self.ms = e0.elapsed_time(e1)

    def close(self, s):
        with torch.cuda.stream(self.g):
            torch.cuda._sleep(self.cycles)
        e = torch.cuda.Event()
        e.record(self.g)
        s.wait_event(e)
        return e


@pytest.fixture(scope="module")
def gate():
    torch.cuda.synchronize()
    g = Gate()
    text = (f"gate: {g.cycles} cycles of torch.cuda._sleep = {g.ms:.1f} ms measured "
            f"({g.cycles_per_ms:.0f} cycles/ms) on {torch.cuda.get_device_name(0)}\n")
    print(text, end="")
    try:
        out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build")
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "test_gpu_streams_gate.txt"), "w") as fh:
            fh.write(text)
    except OSError:
        pass
    assert g.ms > 0.5 * GATE_MS, text
    return g


STREAM_KINDS = ("nonblocking", "high", "low", "legacy")


@pytest.fixture(scope="module")
def streams():
    # torch's side streams are created non-blocking; priority: lower is higher, clamped to the device's range
    return {"nonblocking": torch.cuda.Stream(), "high": torch.cuda.Stream(priority=-100), "low": torch.cuda.Stream(priority=100),
            "legacy": torch.cuda.default_stream()}


# ---------------------------------------------------------------------------------------------------------------------
# buffers and cases
# ---------------------------------------------------------------------------------------------------------------------
def P(t):
    return C.c_void_p(t.data_ptr())


def SP(s):
    return C.c_void_p(s.cuda_stream)


def dev(a, ld=None):
    """numpy vector or (m, n) matrix -> flat device tensor holding it column-major with leading dimension ld (padding 0)."""
    a = np.asarray(a)
    m = a.shape[0]
    n = 1 if a.ndim == 1 else a.shape[1]
    ld = ld or m
    out = np.zeros((n, ld), dtype=a.dtype)
    out[:, :m] = a.reshape(m, n, order="F").T
    return torch.from_numpy(out.ravel()).to(DEV)


def same_bits(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


class Case:
    """One call and its buffers.  ``bufs``: name -> (true content, decoy); the call reads and writes ``work[name]`` (flat device
    tensors) and ``outs`` names its results."""

    def __init__(self, fn, bufs, outs, sync_ok=False):
        self.fn, self.outs, self.sync_ok = fn, tuple(outs), sync_ok
        self.true = {k: v[0] for k, v in bufs.items()}
        self.decoy = {k: v[1] for k, v in bufs.items()}
        self.work = {k: v.clone() for k, v in self.true.items()}
        self.snap = {k: torch.empty_like(self.work[k]) for k in self.outs}

    def load(self, which):
        for k, w in self.work.items():
            w.copy_(which[k])

    def call(self, s):
        self.fn(self.work, SP(s))

    def reference(self, h):
        """Warm-up, then the reference run on the legacy stream; the wide-chain counters of the reference decide whether the call
        may synchronise (dhqr.h point (ii))."""
        leg = torch.cuda.default_stream()
        self.load(self.true)
        self.call(leg)
        torch.cuda.synchronize()
        self.load(self.true)
        c0 = counters(h)
        self.call(leg)
        torch.cuda.synchronize()
        self.delta = {k: v - c0[k] for k, v in counters(h).items()}
        self.sync_ok = self.sync_ok or self.delta["wide_panels"] > 0
        self.ref = {k: self.work[k].clone() for k in self.outs}

    def enqueue(self, s, e=None):
        """On s: true inputs in, the call, snapshots, decoy over every buffer.  Blocks nothing itself; returns whether the gate
        event ``e`` was still pending when the call was made and when it returned."""
        with torch.cuda.stream(s):
            self.load(self.true)
        closed_at_call = e is not None and not e.query()
        self.call(s)
        closed_at_return = e is not None and not e.query()
        with torch.cuda.stream(s):
            for k in self.outs:
                self.snap[k].copy_(self.work[k])
            self.load(self.decoy)
        return closed_at_call, closed_at_return

    def check(self, where):
        for k in self.outs:
            assert same_bits(self.snap[k], self.ref[k]), f"{k} differs bitwise from the ungated legacy-stream run; {where}"


def run_gated(case, gate, s, where):
    case.load(case.decoy)
    torch.cuda.synchronize()
    closed_at_call, closed_at_return = case.enqueue(s, gate.close(s))
    torch.cuda.synchronize()
    assert closed_at_call, f"the gate opened before the call was made (gate too short for this case); {where}"
    if not case.sync_ok:
        assert closed_at_return, f"the call blocked the host until the caller's stream drained; {where}"
    case.check(where)


# ---- case builders ---------------------------------------------------------------------------------------------------
def qr_case(D, h, m, n, nb=0, lda_extra=0, family=FAMILY):
    lda = m + lda_extra
    bufs = {"A": (dev(F.make(family, m, n, 0), lda), dev(F.make(family, m, n, 1), lda)),
            "alpha": (torch.zeros(n, dtype=torch.float64, device=DEV), torch.full((n,), -1.0, dtype=torch.float64, device=DEV))}

    def fn(w, st):
        D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, P(w["A"]), lda, P(w["alpha"]), nb, st)
    return Case(fn, bufs, ("A", "alpha"))


def factor(D, h, A, alpha, m, n, lda, cplx=False):
    if cplx:
        D._lib.call("dhqr_qr_c64", h.raw, m, n, 0, n, P(A), lda, P(alpha), None)
    else:
        D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, P(A), lda, P(alpha), 0, None)
    torch.cuda.synchronize()
    return A, alpha


@pytest.fixture(scope="module")
def fac(D, h):
    """Factorisations of the true and the decoy 2048 x 1024 matrix (real) and 1000 x 300 (complex), made by the module's handle."""
    out = {}
    for seed, key in ((0, "true"), (1, "decoy")):
        A = dev(F.make(FAMILY, M2, N2, seed))
        out[key] = factor(D, h, A, torch.zeros(N2, dtype=torch.float64, device=DEV), M2, N2, M2)
        Ac = dev(F.make_complex("centered", MC, NC, seed))
        out["c" + key] = factor(D, h, Ac, torch.zeros(NC, dtype=torch.complex128, device=DEV), MC, NC, MC, cplx=True)
    return out


def rhs_case(D, h, fac, fn_name, nrhs, ldb_extra=0, cplx=False):
    m, n, pre = (MC, NC, "c") if cplx else (M2, N2, "")
    ldb = m + ldb_extra
    (H, a), (Hd, ad) = fac[pre + "true"], fac[pre + "decoy"]
    bufs = {"H": (H, Hd), "b": (dev(F.rhs(m, nrhs, 0, cplx), ldb), dev(F.rhs(m, nrhs, 1, cplx), ldb))}
    with_alpha = fn_name.startswith(("dhqr_backsolve", "dhqr_solve"))
    if with_alpha:
        bufs["alpha"] = (a, ad)

    def fn(w, st):
        if with_alpha:
            D._lib.call(fn_name, h.raw, m, n, 0, n, P(w["H"]), m, P(w["alpha"]), P(w["b"]), ldb, nrhs, st)
        else:
            D._lib.call(fn_name, h.raw, m, n, 0, n, P(w["H"]), m, P(w["b"]), ldb, nrhs, st)
    return Case(fn, bufs, ("b",))


def householder_block(rows, nbp, seed):
    """rows x nbp reflectors with |v|^2 = 2 (the shape of the packed V the block-reflector hook expects)."""
    g = torch.Generator().manual_seed(seed)
    a, tau = torch.geqrf(torch.rand(rows, nbp, dtype=torch.float64, generator=g))
    V = torch.tril(a, -1) + torch.eye(rows, nbp, dtype=torch.float64)
    return (V * tau.sqrt()).numpy()


def block_reflector_case(D, h, nbp):
    rows, ncols, row_lo = 1000, 100, 0
    nbk = 32 if nbp <= 32 else 128
    bufs = {"V": (dev(householder_block(rows, nbp, 1)), dev(householder_block(rows, nbp, 2))),
            "C": (dev(F.make(FAMILY, rows, ncols, 0)), dev(F.make(FAMILY, rows, ncols, 1))),
            "linv": (torch.zeros(nbk * nbk, dtype=torch.float64, device=DEV), torch.full((nbk * nbk,), -1.0, dtype=torch.float64, device=DEV))}

    def fn(w, st):
        D._lib.call("dhqr_k_block_reflector_f64", h.raw, rows, nbp, P(w["V"]), rows, row_lo, ncols, P(w["C"]), rows, P(w["linv"]), st)
    return Case(fn, bufs, ("C", "linv"))


def panel_case(D, h):
    rows, ncols = 4096, 32
    bufs = {"P": (dev(F.make(FAMILY, rows, ncols, 0)), dev(F.make(FAMILY, rows, ncols, 1))),
            "alpha": (torch.zeros(ncols, dtype=torch.float64, device=DEV), torch.full((ncols,), -1.0, dtype=torch.float64, device=DEV))}

    def fn(w, st):
        D._lib.call("dhqr_k_panel_f64", h.raw, rows, ncols, P(w["P"]), rows, P(w["alpha"]), st)
    return Case(fn, bufs, ("P", "alpha"))


def partialdot_case(D, h, cplx):
    n, i0, i1 = 100_000, 3, 99_991
    dt = torch.complex128 if cplx else torch.float64
    vec = (lambda s: F.rhs(n, 1, s, cplx))
    bufs = {"a": (dev(vec(0)), dev(vec(1))), "b": (dev(vec(2)), dev(vec(3))),
            "out": (torch.zeros(1, dtype=dt, device=DEV), torch.full((1,), -1.0, dtype=dt, device=DEV))}
    name = "dhqr_partialdot_c64" if cplx else "dhqr_partialdot_f64"

    def fn(w, st):
        D._lib.call(name, h.raw, P(w["a"]), P(w["b"]), i0, i1, P(w["out"]), st)
    return Case(fn, bufs, ("out",))


def fill_case(D, h):
    m, n, lda = 1000, 300, 1001
    bufs = {"A": (torch.zeros(n * lda, dtype=torch.float64, device=DEV), dev(F.make(FAMILY, m, n, 1), lda))}

    def fn(w, st):
        D._lib.call("dhqr_fill_uniform_f64", h.raw, 7, 5, 11, m, n, P(w["A"]), lda, st)
    return Case(fn, bufs, ("A",))


def qr_c64_case(D, h):
    bufs = {"A": (dev(F.make_complex("centered", MC, NC, 0)), dev(F.make_complex("centered", MC, NC, 1))),
            "alpha": (torch.zeros(NC, dtype=torch.complex128, device=DEV), torch.full((NC,), -1.0, dtype=torch.complex128, device=DEV))}

    def fn(w, st):
        D._lib.call("dhqr_qr_c64", h.raw, MC, NC, 0, NC, P(w["A"]), MC, P(w["alpha"]), st)
    return Case(fn, bufs, ("A", "alpha"))


# id -> (builder(D, h, fac), options).  The id names the path.
QR_CASES = {
    "qr-default": (lambda D, h, fac: qr_case(D, h, M2, N2), {}),              # look-ahead, wide chain (synchronises)
    "qr-narrow": (lambda D, h, fac: qr_case(D, h, M2, N2), {"wide_panel": 0}),   # look-ahead, 32-column chain, no sync
    "qr-lookahead0": (lambda D, h, fac: qr_case(D, h, M2, N2), {"lookahead": 0}),
    "qr-nb32-lda+1": (lambda D, h, fac: qr_case(D, h, 1000, 300, nb=32, lda_extra=1), {}),
    "qr-nb64-lda+1": (lambda D, h, fac: qr_case(D, h, 1000, 300, nb=64, lda_extra=1), {}),
    "qr-one_panel-300x37": (lambda D, h, fac: qr_case(D, h, 300, 37), {}),
    "qr-nb1-wave-4096x512": (lambda D, h, fac: qr_case(D, h, 4096, 512, nb=1), {}),       # k_unblocked_wave
    "qr-nb1-fused-8400x256": (lambda D, h, fac: qr_case(D, h, 8400, 256, nb=1), {}),      # k_apply1_tma forms the next reflector
    "qr-nb1-column-9000x128": (lambda D, h, fac: qr_case(D, h, 9000, 128, nb=1), {}),     # per-column loop
    "qr-graded12-restart-4099x640": (lambda D, h, fac: qr_case(D, h, 4099, 640, family="graded12"), {}),   # wide chain refuses, redone
}
SOLVE_CASES = {
    "apply_qt-nrhs1-qt_vec1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_qt_f64", 1), {"qt_vec": 1}),
    "apply_qt-nrhs1-qt_vec0": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_qt_f64", 1), {"qt_vec": 0}),
    "apply_qt-nrhs3-ldb+1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_qt_f64", 3, 1), {}),
    "apply_q-nrhs1-qt_vec1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_q_f64", 1), {"qt_vec": 1}),
    "apply_q-nrhs1-qt_vec0": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_q_f64", 1), {"qt_vec": 0}),
    "apply_q-nrhs3-ldb+1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_q_f64", 3, 1), {}),
    "backsolve-nrhs1-bs_wave1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_backsolve_f64", 1), {"bs_wave": 1}),
    "backsolve-nrhs1-bs_wave0": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_backsolve_f64", 1), {"bs_wave": 0}),
    "backsolve-nrhs3-ldb+1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_backsolve_f64", 3, 1), {}),
    "solve-nrhs1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_solve_f64", 1), {}),
    "solve-nrhs3-ldb+1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_solve_f64", 3, 1), {}),
}
OTHER_CASES = {
    "qr_c64": (lambda D, h, fac: qr_c64_case(D, h), {}),
    "apply_qt_c64-nrhs1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_qt_c64", 1, cplx=True), {}),
    "apply_qt_c64-nrhs2": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_apply_qt_c64", 2, cplx=True), {}),
    "backsolve_c64-nrhs1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_backsolve_c64", 1, cplx=True), {}),
    "backsolve_c64-nrhs2": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_backsolve_c64", 2, cplx=True), {}),
    "solve_c64-nrhs1": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_solve_c64", 1, cplx=True), {}),
    "solve_c64-nrhs2": (lambda D, h, fac: rhs_case(D, h, fac, "dhqr_solve_c64", 2, cplx=True), {}),
    "partialdot_c64": (lambda D, h, fac: partialdot_case(D, h, True), {}),
    "partialdot_f64": (lambda D, h, fac: partialdot_case(D, h, False), {}),
    "fill_uniform_f64": (lambda D, h, fac: fill_case(D, h), {}),
    "k_block_reflector-nbp32": (lambda D, h, fac: block_reflector_case(D, h, 32), {}),
    "k_block_reflector-nbp128": (lambda D, h, fac: block_reflector_case(D, h, 128), {}),
    "k_panel-4096x32": (lambda D, h, fac: panel_case(D, h), {}),
}
ALL_CASES = dict(QR_CASES, **SOLVE_CASES, **OTHER_CASES)
# every stream kind for the flagship paths, one non-blocking side stream for the rest
ALL_KINDS = ("qr-default", "qr-narrow", "solve-nrhs1")
PARAMS = [(cid, kind) for cid in ALL_CASES for kind in (STREAM_KINDS if cid in ALL_KINDS else ("nonblocking",))]


@pytest.mark.parametrize("cid,kind", PARAMS, ids=[f"{c}-{k}" for c, k in PARAMS])
def test_gated(D, h, fac, gate, streams, cid, kind):
    build, opts = ALL_CASES[cid]
    case = build(D, h, fac)
    with options(h, **opts):
        case.reference(h)
        run_gated(case, gate, streams[kind], f"{cid} on a {kind} stream (options {opts})")


# ---------------------------------------------------------------------------------------------------------------------
# ordering by the caller across streams: "same stream or ordered by the caller (events)"
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["default", "narrow"])
def test_handoff_qr_then_solve_phases(D, h, gate, path):
    """qr on S1, an event, then apply_qt, backsolve and apply_q on S2 with the same handle, reading the factor qr produced."""
    opts = {} if path == "default" else {"wide_panel": 0}
    m, n = M2, N2
    A0, A1 = dev(F.make(FAMILY, m, n, 0)), dev(F.make(FAMILY, m, n, 1))
    bs = [(dev(F.rhs(m, 1, s)), dev(F.rhs(m, 1, s + 10))) for s in range(3)]
    alpha = torch.zeros(n, dtype=torch.float64, device=DEV)
    A, B = A0.clone(), [b.clone() for b, _ in bs]
    snaps = [torch.empty_like(A), torch.empty_like(alpha)] + [torch.empty_like(b) for b in B]

    def phases(s_qr, s_solve, ev=None):
        D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, P(A), m, P(alpha), 0, SP(s_qr))
        with torch.cuda.stream(s_qr):
            snaps[0].copy_(A)
            snaps[1].copy_(alpha)
        if ev is not None:
            ev.record(s_qr)
            s_solve.wait_event(ev)
        D._lib.call("dhqr_apply_qt_f64", h.raw, m, n, 0, n, P(A), m, P(B[0]), m, 1, SP(s_solve))
        D._lib.call("dhqr_backsolve_f64", h.raw, m, n, 0, n, P(A), m, P(alpha), P(B[1]), m, 1, SP(s_solve))
        D._lib.call("dhqr_apply_q_f64", h.raw, m, n, 0, n, P(A), m, P(B[2]), m, 1, SP(s_solve))

    def reset(which):
        A.copy_(A0 if which == 0 else A1)
        alpha.fill_(-1.0)
        for b, (bt, bd) in zip(B, bs):
            b.copy_(bt if which == 0 else bd)

    leg = torch.cuda.default_stream()
    with options(h, **opts):
        for _ in range(2):                      # warm-up, then the reference
            reset(0)
            phases(leg, leg)
            torch.cuda.synchronize()
        ref = [A.clone(), alpha.clone()] + [b.clone() for b in B]
        reset(1)
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        e = gate.close(s1)
        with torch.cuda.stream(s1):
            A.copy_(A0)
            for b, (bt, _) in zip(B, bs):
                b.copy_(bt)
        phases(s1, s2, torch.cuda.Event())
        closed = not e.query()
        with torch.cuda.stream(s2):
            for snap, b in zip(snaps[2:], B):
                snap.copy_(b)
            A.copy_(A1)
            alpha.fill_(-1.0)
        torch.cuda.synchronize()
    if path == "narrow":
        assert closed, "a call blocked the host while the caller's streams were gated"
    for name, got, want in zip(("H", "alpha", "Q'b", "R\\b", "Qb"), snaps, ref):
        assert same_bits(got, want), f"{name} differs bitwise from the serial legacy-stream run (qr on S1, solve phases on S2, {path})"


def test_handoff_solve_then_qr_overwrites_factor(D, h, fac, gate):
    """A solve on S2, then a new narrow qr on S1 (ordered after the solve by an event) that factors a new matrix in the very
    buffer the solve reads."""
    m, n = M2, N2
    (Ht, at), _ = fac["true"], fac["decoy"]
    Anew = dev(F.make(FAMILY, m, n, 2))
    b0 = dev(F.rhs(m, 1, 0))
    Hbuf, abuf, b = Ht.clone(), at.clone(), b0.clone()
    snaps = [torch.empty_like(b), torch.empty_like(Hbuf), torch.empty_like(abuf)]

    def seq(s_solve, s_qr, ev=None):
        D._lib.call("dhqr_solve_f64", h.raw, m, n, 0, n, P(Hbuf), m, P(abuf), P(b), m, 1, SP(s_solve))
        with torch.cuda.stream(s_solve):
            snaps[0].copy_(b)
        if ev is not None:
            ev.record(s_solve)
            s_qr.wait_event(ev)
        with torch.cuda.stream(s_qr):
            Hbuf.copy_(Anew)
        D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, P(Hbuf), m, P(abuf), 0, SP(s_qr))
        with torch.cuda.stream(s_qr):
            snaps[1].copy_(Hbuf)
            snaps[2].copy_(abuf)

    leg = torch.cuda.default_stream()
    with options(h, wide_panel=0):
        for _ in range(2):
            Hbuf.copy_(Ht), abuf.copy_(at), b.copy_(b0)
            seq(leg, leg)
            torch.cuda.synchronize()
        ref = [t.clone() for t in snaps]
        Hbuf.fill_(0.5), abuf.fill_(-1.0), b.fill_(0.25)
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        e = gate.close(s2)
        with torch.cuda.stream(s2):
            Hbuf.copy_(Ht), abuf.copy_(at), b.copy_(b0)
        seq(s2, s1, torch.cuda.Event())
        closed = not e.query()
        torch.cuda.synchronize()
    assert closed, "a call blocked the host while the caller's streams were gated"
    for name, got, want in zip(("x", "H of the new matrix", "alpha of the new matrix"), snaps, ref):
        assert same_bits(got, want), f"{name} differs bitwise from the serial legacy-stream run (solve on S2, then qr on S1)"


# ---------------------------------------------------------------------------------------------------------------------
# the Python layer picks up torch's current stream
# ---------------------------------------------------------------------------------------------------------------------
def test_python_layer_on_current_stream(D, h, gate):
    """qr_, apply_qt_, apply_q_, backsolve_, solve_householder_, ldiv and the one-rank ColumnBlockMatrix under
    torch.cuda.stream(S): they return with S gated (their torch.zeros / clone calls land on S too) and give the C-ABI's bits."""
    m, n = M2, N2
    A0, b0 = dev(F.make(FAMILY, m, n, 0)), dev(F.rhs(m, 1, 0))
    A, Acb = torch.empty_like(A0), torch.empty_like(A0)
    B = [torch.empty_like(b0) for _ in range(4)]
    dA = A.view(n, m).t()
    dAcb = Acb.view(n, m).t()
    leg = torch.cuda.default_stream()

    # the C-ABI reference, on the legacy stream
    with options(h, wide_panel=0):
        Hr, ar = A0.clone(), torch.zeros(n, dtype=torch.float64, device=DEV)
        D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, P(Hr), m, P(ar), 0, SP(leg))
        ref = {"H": Hr, "alpha": ar}
        for key, fn, with_alpha in (("qtb", "dhqr_apply_qt_f64", False), ("qb", "dhqr_apply_q_f64", False),
                                    ("rb", "dhqr_backsolve_f64", True), ("x", "dhqr_solve_f64", True)):
            r = b0.clone()
            if with_alpha:
                D._lib.call(fn, h.raw, m, n, 0, n, P(Hr), m, P(ar), P(r), m, 1, SP(leg))
            else:
                D._lib.call(fn, h.raw, m, n, 0, n, P(Hr), m, P(r), m, 1, SP(leg))
            ref[key] = r
        torch.cuda.synchronize()

    s = torch.cuda.Stream()

    def layer():
        with torch.cuda.stream(s):
            A.copy_(A0)
            Acb.copy_(A0)
            for b in B:
                b.copy_(b0)
            H = D.qr_(dA, handle=h)
            D.apply_qt_(B[0], dA, handle=h)
            D.apply_q_(B[1], dA, handle=h)
            D.backsolve_(B[2], dA, H.α, handle=h)
            D.solve_householder_(B[3], dA, H.α, handle=h)
            x = D.ldiv(H, b0)
            Hcb = D.qr_(D.ColumnBlockMatrix(dAcb, n, 0, handle=h))
            xcb = D.ldiv(Hcb, b0)
            return H, x, Hcb, xcb

    with options(h, wide_panel=0):
        layer()                                 # warm-up: workspace, and blocks in torch's cache for S
        torch.cuda.synchronize()
        A.fill_(0.5), Acb.fill_(0.5)
        for b in B:
            b.fill_(0.25)
        torch.cuda.synchronize()
        e = gate.close(s)
        H, x, Hcb, xcb = layer()
        closed = not e.query()
        torch.cuda.synchronize()
    assert closed, "a Python-layer call blocked the host while torch's current stream was gated"
    got = {"H": A, "alpha": H.α, "qtb": B[0], "qb": B[1], "rb": B[2][:n], "x": B[3][:n], "ldiv": x,
           "ColumnBlockMatrix H": Acb, "ColumnBlockMatrix alpha": Hcb.α, "ColumnBlockMatrix ldiv": xcb}
    want = {"H": ref["H"], "alpha": ref["alpha"], "qtb": ref["qtb"], "qb": ref["qb"], "rb": ref["rb"][:n], "x": ref["x"][:n],
            "ldiv": ref["x"][:n], "ColumnBlockMatrix H": ref["H"], "ColumnBlockMatrix alpha": ref["alpha"],
            "ColumnBlockMatrix ldiv": ref["x"][:n]}
    for k in got:
        assert same_bits(got[k].contiguous(), want[k].contiguous()), f"{k} differs bitwise from the C-ABI on the legacy stream"


# ---------------------------------------------------------------------------------------------------------------------
# a fresh handle's first calls while the legacy default stream is busy
# ---------------------------------------------------------------------------------------------------------------------
def test_fresh_handle_first_calls_with_busy_default_stream(D, h, gate):
    """A fresh handle zero-fills the workspace its first calls hand data through (back-substitution cells, nb = 1 wave flags,
    the Q'b ticket, panel counters, wide-chain control words).  Those fills must be ordered on the caller's stream: with the
    legacy stream gated and the calls on a non-blocking stream, a fill on the legacy stream would land after the kernels that
    need it, and recycled memory from an earlier handle (holding its tags) would be read as fresh data."""
    m, n = MF, NF
    mats = {s: dev(F.make(FAMILY, m, n, s)) for s in (0, 1, 2, 3)}
    rhs = {s: dev(F.rhs(m, 1, s)) for s in (0, 1)}
    # factorisations made by the module handle: the backsolve's input (seed 0) and the throwaway handle's (seed 1)
    facs = {s: factor(D, h, mats[s].clone(), torch.zeros(n, dtype=torch.float64, device=DEV), m, n, m) for s in (0, 1)}

    def sequence(hd, s, data):
        """backsolve, nb = 1 qr, nrhs = 1 apply_qt, narrow qr: the first call of each kind on a handle.  Same shapes
        throughout, so no buffer grows (no cudaFree, which would drain the legacy stream) once the first call sized them."""
        (Hf, af), b1, Aq1, b2, Aq2, outs = data
        st = SP(s)
        D._lib.call("dhqr_backsolve_f64", hd.raw, m, n, 0, n, P(Hf), m, P(af), P(b1), m, 1, st)
        D._lib.call("dhqr_qr_f64", hd.raw, m, n, 0, n, P(Aq1), m, P(outs[0]), 1, st)
        D._lib.call("dhqr_apply_qt_f64", hd.raw, m, n, 0, n, P(Hf), m, P(b2), m, 1, st)
        hd.set_option("wide_panel", 0)
        D._lib.call("dhqr_qr_f64", hd.raw, m, n, 0, n, P(Aq2), m, P(outs[1]), 0, st)

    def data(fseed, bseed, a1, a2):
        return (facs[fseed], rhs[bseed].clone(), mats[a1].clone(), rhs[bseed].clone(), mats[a2].clone(),
                [torch.zeros(n, dtype=torch.float64, device=DEV) for _ in range(2)])

    leg = torch.cuda.default_stream()
    # reference: the module handle (default options, like a fresh one), ungated
    ref = data(0, 0, 2, 3)
    with options(h, wide_panel=1):
        sequence(h, leg, ref)
    torch.cuda.synchronize()
    # a throwaway handle runs the same sequence on other data, and leaves its tags in memory it hands back
    t = D.Handle(0)
    sequence(t, leg, data(1, 1, 3, 2))
    torch.cuda.synchronize()
    t.close()
    # the fresh handle: same inputs as the reference, first calls on a non-blocking stream while the legacy stream is gated
    got = data(0, 0, 2, 3)
    torch.cuda.synchronize()
    fresh = D.Handle(0)
    try:
        s = torch.cuda.Stream()
        gate.close(leg)
        sequence(fresh, s, got)
        torch.cuda.synchronize()
    finally:
        fresh.close()
    names = ("x (backsolve, first call)", "Q'b (apply_qt)", "H (nb = 1 qr)", "H (narrow qr)", "alpha (nb = 1 qr)",
             "alpha (narrow qr)")
    for name, a, b in zip(names, (got[1], got[3], got[2], got[4], got[5][0], got[5][1]),
                          (ref[1], ref[3], ref[2], ref[4], ref[5][0], ref[5][1])):
        assert same_bits(a, b), f"{name} of a fresh handle differs bitwise from the reference while the default stream was busy"


# ---------------------------------------------------------------------------------------------------------------------
# counters, read the documented way: after synchronising the stream of the calls
# ---------------------------------------------------------------------------------------------------------------------
def test_counters_after_stream_sync(D, h, gate):
    narrow, wide = qr_case(D, h, M2, N2), qr_case(D, h, M2, N2)
    with options(h, wide_panel=0):
        narrow.reference(h)
    wide.reference(h)
    assert narrow.delta["panels_fast"] + narrow.delta["panels_fallback"] == N2 // 32 and narrow.delta["wide_panels"] == 0
    assert wide.delta["wide_panels"] == N2 // 128 and wide.delta["wide_redone"] == 0
    narrow.load(narrow.decoy), wide.load(wide.decoy)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    c0 = counters(h)
    gate.close(s)
    with options(h, wide_panel=0):
        narrow.enqueue(s)
    wide.enqueue(s)
    s.synchronize()
    c1 = counters(h)
    for k in COUNTERS:
        assert c1[k] - c0[k] == narrow.delta[k] + wide.delta[k], \
            f"{k}: {c1[k] - c0[k]} after the stream's synchronisation, the gated calls ran {narrow.delta[k] + wide.delta[k]}"
    narrow.check("narrow qr, counters")
    wide.check("wide qr, counters")


# ---------------------------------------------------------------------------------------------------------------------
# host entry points: no stream of their own to take, so none of the caller's may hold them up
# ---------------------------------------------------------------------------------------------------------------------
def test_host_entry_with_gated_legacy_stream(D, h, gate):
    m, n = 4096, 2048                           # several upload chunks at the default host_chunk: the pipelined path
    A0 = np.asfortranarray(F.make(FAMILY, m, n, 0))
    b0 = F.rhs(m, 1, 0)

    def pinned(n):
        t = torch.empty(n, dtype=torch.float64, pin_memory=True)
        return t, t.numpy()

    (tA, vA), (ta, va), (tb, vb), (tx, vx) = pinned(A0.size), pinned(n), pinned(m), pinned(n)
    vb[:] = b0

    def run():
        vA[:] = A0.ravel(order="F")
        va[:], vx[:] = 0.0, 0.0
        D._lib.call("dhqr_qr_host_f64", h.raw, m, n, P(tA), m, P(ta), 0)
        D._lib.call("dhqr_ldiv_host_f64", h.raw, m, n, P(tA), m, P(ta), P(tb), P(tx))
        return vA.copy(), va.copy(), vx.copy()

    run()                                       # warm-up
    ref = run()
    torch.cuda.synchronize()
    gate.close(torch.cuda.default_stream())
    got = run()
    torch.cuda.synchronize()
    for name, a, b in zip(("H", "alpha", "x"), got, ref):
        assert a.tobytes() == b.tobytes(), f"{name} of the host entry differs bitwise while the legacy stream was gated"
