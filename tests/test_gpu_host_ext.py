"""The pipelined host entry (dhqr_qr_host_f64, dhqr_ldiv_host_f64) held to the extended-precision rule of ext_rule.py, with the
host matrix in pinned memory so that the pipeline really runs (run with -m gpu on an H100).

With pageable memory every chunk copy blocks the host and the factorisation starts after the last one (DESIGN §9), so every
upload event has fired before any kernel runs.  Here every host operand is a page-locked torch buffer viewed column-major:
the later chunks are still on the link while the first panels are factored, join the window through a catch-up on one of
the cu_streams, and finished panels travel back while later ones are factored.  Each case takes its plan from the product's
planner (plan_host_upload) and asserts that the plan is windowed where it means to exercise the pipeline.

    families x plans      every non-NaN family at 2048 x 1024 under deadline joins (host_chunk 128, 1 GB/s: the chunk holding
                          panel p joins at step p - 3), early joins (100000 GB/s: steps 0 and 1) and a 640-column first upload
                          (host_chunk 384, host_first 640), each with 1 and 3 catch-up streams: V, R, bwd, orth, and x from
                          dhqr_ldiv_host_f64
    panel widths          nb = 32 / 64 / 96 at 2304 x 1152; a 76-column last panel (3000 x 1100); m = 4099 with host lda = m + 3
                          (padded device ldd); 1152 x 1152, where the late catch-ups run on short windows
    overlapping shape     16384 x 2048 at the default plan and at host_chunk 128: the first 1024 columns to the rule, all 2048
                          to bwd / orth, every setting twice and bitwise equal
    function of the plan  runs grouped by the planner's (bounds, join) over catch-up streams, model parameters that give the
                          same plan, host_trace and pinned / pageable: bitwise equal within a group; host_chunk = 0 and nb = 1
                          bitwise equal to the device entry, dhqr_ldiv_host_f64 bitwise equal to dhqr_solve_f64
    the driver's joins    host_trace's "joins at step J (planned P)": J == P and the plan of plan_host_upload, chunk by chunk
    refusals              a nearly rank-deficient panel f at 3000 x 1408 (11 panels): inside the first upload, the first panel
                          of a late chunk, behind the catch-ups of later chunks, the last panel, and two refusals (three passes)
    zero columns          the zero column in a late chunk: the fp64 oracle's NaN pattern, the leading columns to the rule
    Python layer          qr_ on a numpy view of a pinned buffer + ldiv: bitwise the raw C-ABI calls, b untouched

Overlap at 16384 x 2048 (a 268 MB upload; the default plan sends columns 384 .. 2047 in four chunks behind the first), measured
with host_trace = 1 on an H100 80GB HBM3 (SXM, 700 W): the last chunk was on the device 6.1 ms after the factorisation started,
step 0's panel 0.4 ms after it, so the uploads overlap the chain.  The long double reference of the 1024-column prefix (with its
fp64 twin) took 10 to 13 s on 16 CPU cores (two runs).  The link speed differs between parts (SXM, PCIe), so the overlap is asserted where it
is measured, not assumed.

A table of err_gpu / max(err_fp64_oracle, FLOOR) per case x family is written to build/test_gpu_host_ext_ratios.md.
"""
import contextlib
import ctypes as C
import os
import re
import time

import numpy as np
import pytest
import torch

import matrix_families as F
from ext_rule import COUNTERS, Ref, Table, backward_error, counters, digest, factor_checks, nrm, orth_error, TOL_BWD, TOL_ORTH

pytestmark = pytest.mark.gpu

# the host options and their defaults; all but host_chunk can be set and not read back, so a block puts the defaults back
HOST_DEFAULTS = dict(host_chunk=512, host_first=0, host_h2d_gbs=50, host_tflops=27, host_chain_us=300, host_cu_streams=3, host_trace=0)
DEADLINE = dict(host_chunk=128, host_h2d_gbs=1)           # every chunk joins one step before the chain reaches into it

TABLE = Table("test_gpu_host_ext_ratios.md")
NOTES = []


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


@pytest.fixture(scope="module")
def h(D):
    hh = D.Handle(0)                                       # its own handle: no option state leaks in or out
    yield hh
    hh.close()


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    TABLE.write()
    if NOTES and TABLE.ratios:
        path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", TABLE.name)
        try:
            with open(path, "a") as fh:
                fh.write("\n" + "\n".join(f"- {s}" for s in NOTES) + "\n")
        except OSError:
            pass


# ---------------------------------------------------------------------------------------------------------------------
# host operands and calls
# ---------------------------------------------------------------------------------------------------------------------
def pinned(A0, lda=None):
    """A page-locked, column-major copy of A0 with leading dimension lda: (the buffer, its (m, n) view)."""
    m, n = A0.shape[0], (A0.shape[1] if A0.ndim == 2 else 1)
    buf = torch.empty((n, lda or m), dtype=torch.float64).pin_memory()
    view = buf.t()[:m]
    view.copy_(torch.from_numpy(np.reshape(A0, (m, n), order="F")))
    return buf, view


@contextlib.contextmanager
def host_options(h, **kw):
    """Set the host options for a block (the rest at their defaults) and yield the whole setting; the defaults afterwards."""
    setting = dict(HOST_DEFAULTS, **kw)
    try:
        for k, v in setting.items():
            h.set_option(k, v)
        yield setting
    finally:
        for k, v in HOST_DEFAULTS.items():
            h.set_option(k, v)


def plan(D, o, m, n, nb):
    """The planner's (bounds, join) for the host options o."""
    return D.plan_host_upload(m, n, nb or 128, chunk=o["host_chunk"], first=o["host_first"], h2d_gbs=o["host_h2d_gbs"],
                              tflops=o["host_tflops"], chain_us=o["host_chain_us"])


def host_qr(D, h, A0, nb=0, lda=None, pin=True):
    """dhqr_qr_host_f64 on a pinned (or pageable numpy) copy of A0 -> (H, alpha, counter deltas, note)."""
    m, n = A0.shape
    lda = lda or m
    if pin:
        buf, view = pinned(A0, lda)
        alpha = torch.empty(n, dtype=torch.float64).pin_memory().fill_(np.nan)
        pa, pal = view.data_ptr(), alpha.data_ptr()
    else:
        buf = np.zeros((lda, n), order="F")
        buf[:m] = A0
        view, alpha = buf[:m], np.full(n, np.nan)
        pa, pal = buf.ctypes.data, alpha.ctypes.data
    c0 = counters(h)
    D._lib.call("dhqr_qr_host_f64", h.raw, m, n, C.c_void_p(pa), lda, C.c_void_p(pal), nb)
    c1 = counters(h)
    H = np.array(view.numpy() if pin else view, order="F")
    note = "counters " + ", ".join(f"{k} {c0[k]}->{c1[k]}" for k in COUNTERS)
    return H, (alpha.numpy() if pin else alpha).copy(), {k: c1[k] - c0[k] for k in COUNTERS}, note


def host_ldiv(D, h, H, alpha, b0):
    """dhqr_ldiv_host_f64 with every operand pinned; b must come back untouched."""
    m, n = H.shape
    _, Hp = pinned(H)
    _, ap = pinned(alpha)
    _, bp = pinned(b0)
    x = torch.full((n,), np.nan, dtype=torch.float64).pin_memory()
    D._lib.call("dhqr_ldiv_host_f64", h.raw, m, n, C.c_void_p(Hp.data_ptr()), m, C.c_void_p(ap.data_ptr()),
                C.c_void_p(bp.data_ptr()), C.c_void_p(x.data_ptr()))
    assert np.array_equal(bp.numpy()[:, 0], b0), "dhqr_ldiv_host_f64 wrote to b"
    return x.numpy().copy()


def hold(path, ref, H, alpha, note, x=None, all_cols=False):
    """The rule on V and R (leading ref.k columns), the absolute bounds, and on x where the family is solvable."""
    gpu, absolute = factor_checks(path, ref, H, alpha, note)
    e64 = dict(ref.e64)
    if x is not None:
        gpu["x"] = nrm(x - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])
        e64["x"] = nrm(ref.x64[:, 0] - ref.x_e[:, 0]) / nrm(ref.x_e[:, 0])
    if all_cols:
        absolute["bwd all"] = (backward_error(ref.A, H, alpha), TOL_BWD)
        absolute["orth all"] = (orth_error(H, ref.n), TOL_ORTH)
    TABLE.check(path, ref, gpu, e64, absolute, note)


def windowed(bounds, join):
    assert len(bounds) > 2, f"the plan is a single upload: {bounds}"
    return f"plan {list(zip(bounds[:-1], join))}"


# ---------------------------------------------------------------------------------------------------------------------
# 1. every family under deadline joins, early joins and a wide first upload, with 1 and 3 catch-up streams
# ---------------------------------------------------------------------------------------------------------------------
PLANS = {  # name -> (options, first column of the second chunk)
    "c128 deadline": (DEADLINE, 384),
    "c128 early": (dict(host_chunk=128, host_h2d_gbs=100000), 384),
    "c384 first640": (dict(host_chunk=384, host_h2d_gbs=3, host_first=640), 640),
}


@pytest.mark.parametrize("family", [f for f in F.FAMILIES if f not in F.NAN_FAMILIES])
def test_families_under_every_plan(D, h, oracle, coracle, family):
    m, n = 2048, 1024
    ref = Ref(coracle, oracle, family, m, n)
    for name, (opts, first) in PLANS.items():
        for cu in (1, 3):
            with host_options(h, host_cu_streams=cu, **opts) as o:
                bounds, join = plan(D, o, m, n, 0)
                H, a, _, note = host_qr(D, h, ref.A)
            note += "; " + windowed(bounds, join)
            assert bounds[1] == first, f"the first upload should end at column {first}; {note}"
            x = host_ldiv(D, h, H, a, ref.b[:, 0].copy()) if ref.solve else None
            hold(f"{name} cu{cu}", ref, H, a, note, x)


# ---------------------------------------------------------------------------------------------------------------------
# 2. narrow panels and ragged shapes, deadline joins
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["normal", "graded12", "colscale", "kahan"])
def test_panel_widths(D, h, oracle, coracle, family):
    m, n = 2304, 1152
    ref = Ref(coracle, oracle, family, m, n)
    for nb in (32, 64, 96):
        with host_options(h, **DEADLINE) as o:
            bounds, join = plan(D, o, m, n, nb)
            H, a, _, note = host_qr(D, h, ref.A, nb)
        note += "; " + windowed(bounds, join)
        x = host_ldiv(D, h, H, a, ref.b[:, 0].copy()) if ref.solve else None
        hold(f"nb{nb} deadline", ref, H, a, note, x)


RAGGED = {  # name -> (m, n, extra rows of the host lda)
    "3000x1100 (last panel 76)": (3000, 1100, 0),
    "4099x1408 lda+3": (4099, 1408, 3),
    "1152x1152": (1152, 1152, 0),
}


@pytest.mark.parametrize("family", ["normal", "colscale"])
@pytest.mark.parametrize("shape", list(RAGGED))
def test_ragged_shapes(D, h, oracle, coracle, shape, family):
    m, n, extra = RAGGED[shape]
    ref = Ref(coracle, oracle, family, m, n)
    for cu in (1, 3):
        with host_options(h, host_cu_streams=cu, **DEADLINE) as o:
            bounds, join = plan(D, o, m, n, 0)
            H, a, _, note = host_qr(D, h, ref.A, lda=m + extra)
        note += "; " + windowed(bounds, join)
        x = host_ldiv(D, h, H, a, ref.b[:, 0].copy()) if ref.solve else None
        hold(f"{shape} cu{cu}", ref, H, a, note, x)


# ---------------------------------------------------------------------------------------------------------------------
# 3. a shape at which the uploads overlap the factorisation
# ---------------------------------------------------------------------------------------------------------------------
TRACE_CHUNK = re.compile(r"\[dhqr host\] chunk at column\s+(\d+): uploaded\s+(-?[\d.]+) ms, joins at step\s+(\d+) \(planned\s+(\d+)\)")
TRACE_STEP = re.compile(r"\[dhqr host\] step\s+(\d+): panel\s+(-?[\d.]+)")
TRACE_PLAN = re.compile(r"\[dhqr host\] upload chunks \(first column : join step\):((?: \d+:\d+)+)")


def test_overlapping_shape(D, h, oracle, coracle, capfd):
    m, n, k = 16384, 2048, 1024
    t = time.perf_counter()
    ref = Ref(coracle, oracle, "normal", m, n, k=k, solve=False)
    NOTES.append(f"extended reference of the {m} x {k} prefix (with its fp64 twin): {time.perf_counter() - t:.1f} s on the CPU")
    runs = {}
    for name, opts in {"default": {}, "c128": dict(host_chunk=128)}.items():
        for cu in (1, 3):
            with host_options(h, host_cu_streams=cu, **opts) as o:
                bounds, join = plan(D, o, m, n, 0)
                H, a, _, note = host_qr(D, h, ref.A)
                H2, a2, _, _ = host_qr(D, h, ref.A)
            note += "; " + windowed(bounds, join)
            # the prefix spans the first upload and at least two late chunks, one of them with catch-up work
            assert bounds[1] < k and sum(1 for c in bounds[1:-1] if c < k) >= 2 and max(j for c, j in zip(bounds, join) if c < k) > 0, note
            runs[(name, cu)] = digest(H, a)
            assert runs[(name, cu)] == digest(H2, a2), f"two runs differ bitwise; {name} cu{cu}; {note}"
            hold(f"{m}x{n} {name} cu{cu}", ref, H, a, note, all_cols=True)
            del H, H2
    capfd.readouterr()
    with host_options(h, host_trace=1, host_cu_streams=3) as o:
        bounds, join = plan(D, o, m, n, 0)
        H, a, _, _ = host_qr(D, h, ref.A)
    err = capfd.readouterr().err
    assert digest(H, a) == runs[("default", 3)], "host_trace = 1 changed the result"
    up = [float(g[1]) for g in TRACE_CHUNK.findall(err)]
    step0 = [float(g[1]) for g in TRACE_STEP.findall(err) if int(g[0]) == 0]
    assert up and step0, err
    NOTES.append(f"{m} x {n} default plan {bounds}: last chunk uploaded {max(up):.2f} ms, step 0 panel {step0[0]:.2f} ms "
                 f"(after the factorisation started)")
    assert max(up) > step0[0], f"no upload overlaps the chain at {m} x {n}:\n{err}"


# ---------------------------------------------------------------------------------------------------------------------
# 4. the result is a function of the plan
# ---------------------------------------------------------------------------------------------------------------------
def same_plan_models(D, m, n, chunk):
    """Two (h2d_gbs, tflops, chain_us) triples with different link speeds that the planner maps to the same windowed plan."""
    seen = {}
    for gbs in (1, 2, 3, 5, 10, 20):
        for tf in (10, 27, 60):
            for chain in (100, 300, 1000):
                b, j = D.plan_host_upload(m, n, 128, chunk=chunk, h2d_gbs=gbs, tflops=tf, chain_us=chain)
                if len(b) <= 2:
                    continue
                for other in seen.get((tuple(b), tuple(j)), []):
                    if other[0] != gbs and max(j) > 1:
                        return other, (gbs, tf, chain)
                seen.setdefault((tuple(b), tuple(j)), []).append((gbs, tf, chain))
    return None


def test_result_is_a_function_of_the_plan(D, h, capfd):
    m, n = 2048, 1024
    A0 = F.make("normal", m, n)
    pair = same_plan_models(D, m, n, 128)
    assert pair, "no two model settings with different link speeds give the same plan"
    models = list(pair) + [(100000, 27, 300)]
    groups = {}
    for gbs, tf, chain in models:
        for cu in (1, 2, 3):
            for trace in (0, 1):
                for pin in (True, False):
                    with host_options(h, host_chunk=128, host_h2d_gbs=gbs, host_tflops=tf, host_chain_us=chain, host_cu_streams=cu,
                                      host_trace=trace) as o:
                        key = tuple(map(tuple, plan(D, o, m, n, 0)))
                        H, a, _, _ = host_qr(D, h, A0, pin=pin)
                    groups.setdefault(key, {})[(gbs, tf, chain, cu, trace, pin)] = digest(H, a)
    capfd.readouterr()
    assert len(groups) >= 2 and all(len(k[0]) > 2 for k in groups)
    assert sum(len(g) for g in groups.values() if any(s[:3] == pair[0] for s in g) and any(s[:3] == pair[1] for s in g)) == 24
    for key, g in groups.items():
        ref_setting, ref_digest = next(iter(g.items()))
        for s, d in g.items():
            assert d == ref_digest, f"plan {key}: (gbs, tflops, chain_us, cu_streams, trace, pinned) {s} differs bitwise from {ref_setting}"

    # one upload: bitwise the device entry on a device copy; dhqr_ldiv_host_f64 bitwise dhqr_solve_f64 on the same (H, alpha)
    b0 = F.rhs(m)
    with host_options(h, host_chunk=0) as o:
        assert len(plan(D, o, m, n, 0)[0]) == 2
        H, a, _, _ = host_qr(D, h, A0)
    dA = D.to_colmajor(A0, "cuda:0")
    st = D.qr_(dA, handle=h)
    torch.cuda.synchronize()
    assert digest(H, a) == digest(dA.cpu().numpy(), st.α.cpu().numpy()), "host_chunk = 0 differs bitwise from dhqr_qr_f64"
    x = host_ldiv(D, h, H, a, b0)
    dH = D.to_colmajor(H, "cuda:0")
    db = torch.from_numpy(b0.copy()).cuda()
    D.solve_householder_(db, dH, torch.from_numpy(a).cuda(), handle=h)
    assert digest(x) == digest(db[:n].cpu().numpy()), "dhqr_ldiv_host_f64 differs bitwise from dhqr_solve_f64"

    # nb = 1 (unblocked; one upload whatever the chunk option) through the host: bitwise the device nb = 1
    A1 = np.asfortranarray(A0[:, :256])
    with host_options(h, **DEADLINE) as o:
        H1, a1, _, _ = host_qr(D, h, A1, nb=1)
    dA1 = D.to_colmajor(A1, "cuda:0")
    st1 = D.qr_(dA1, nb=1, handle=h)
    torch.cuda.synchronize()
    assert digest(H1, a1) == digest(dA1.cpu().numpy(), st1.α.cpu().numpy()), "host nb = 1 differs bitwise from device nb = 1"


# ---------------------------------------------------------------------------------------------------------------------
# 5. the driver joins every chunk at the step the planner named
# ---------------------------------------------------------------------------------------------------------------------
JOIN_CASES = {  # name -> (m, n, nb, options, first column of the second chunk or None)
    "2048x1024 deadline": (2048, 1024, 0, DEADLINE, 384),
    "2048x1024 early": (2048, 1024, 0, dict(host_chunk=128, host_h2d_gbs=100000), 384),
    "3000x1408 c512 first640": (3000, 1408, 0, dict(host_chunk=512, host_first=640), 640),
    "2048x1024 c384 first640 3GB/s": (2048, 1024, 0, dict(host_chunk=384, host_h2d_gbs=3, host_first=640), 640),
    "2048x1024 nb64 deadline": (2048, 1024, 64, DEADLINE, 192),
    "2304x1152 nb32 3GB/s": (2304, 1152, 32, dict(host_chunk=128, host_h2d_gbs=3), 96),
    "16384x2048 default": (16384, 2048, 0, {}, 384),
}


@pytest.mark.parametrize("case", list(JOIN_CASES))
def test_the_driver_joins_where_the_plan_says(D, h, capfd, case):
    m, n, nb, opts, first = JOIN_CASES[case]
    A0 = F.make("normal", m, n)
    with host_options(h, host_trace=1, **opts) as o:
        bounds, join = plan(D, o, m, n, nb)
        capfd.readouterr()
        host_qr(D, h, A0, nb)
        err = capfd.readouterr().err
    note = windowed(bounds, join)
    assert bounds[1] == first, f"the first upload should end at column {first}; {note}"
    hdr = TRACE_PLAN.search(err)
    assert hdr, err
    assert [tuple(map(int, s.split(":"))) for s in hdr.group(1).split()] == list(zip(bounds[:-1], join)), f"{hdr.group(0)}; {note}"
    got = [(int(g[0]), int(g[2]), int(g[3])) for g in TRACE_CHUNK.findall(err)]
    assert [c for c, _, _ in got] == bounds[1:-1], f"chunks the driver joined: {got}; {note}"
    assert [p for _, _, p in got] == join[1:], f"planned steps the driver saw: {got}; {note}"
    assert all(j == p for _, j, p in got), f"a chunk joined at another step than planned: {got}; {note}"


# ---------------------------------------------------------------------------------------------------------------------
# 6. refused wide panels at every position of the plan
# ---------------------------------------------------------------------------------------------------------------------
REFUSED = {  # name -> refused panels; 3000 x 1408 at host_chunk 128: first upload = panels 0..2, then one panel per chunk
    "f0": (0,),              # inside the first upload
    "f2": (2,),
    "f3": (3,),              # the first panel of a late chunk
    "f5": (5,),              # under deadline joins the chunks at 1152 and 1280 join at steps 6 and 7: V_5 rides their catch-ups
    "f10": (10,),            # the last panel: the second pass is serial
    "f2+f6": (2, 6),         # three passes
}


def nearly_deficient(m, n, panels):
    A0 = F.make("normal", m, n)
    rng = np.random.default_rng([m, n, 15])
    for f in panels:                                     # one column of panel f = another column of it + 1e-11 noise
        A0[:, 128 * f + 70] = A0[:, 128 * f + 10] + 1e-11 * rng.standard_normal(m)
    return A0


@pytest.mark.parametrize("case", list(REFUSED))
def test_refusal_positions(D, h, oracle, coracle, case):
    m, n = 3000, 1408
    A0 = nearly_deficient(m, n, REFUSED[case])
    ref = Ref(coracle, oracle, f"refused {case}", m, n, solve=False, A=A0)
    for gbs in (1, 100000):
        for cu in (1, 3):
            with host_options(h, host_chunk=128, host_h2d_gbs=gbs, host_cu_streams=cu) as o:
                bounds, join = plan(D, o, m, n, 0)
                H, a, delta, note = host_qr(D, h, A0)
                Hp, ap, _, _ = host_qr(D, h, A0, pin=False)
            note += f"; {gbs} GB/s, cu{cu}; " + windowed(bounds, join)
            assert delta["wide_redone"] == len(REFUSED[case]), f"refused panels {REFUSED[case]}; {note}"
            hold(f"{gbs} GB/s cu{cu}", ref, H, a, note)
            # the host buffer holds the last pass, not panels mirrored back by an earlier one
            assert digest(H, a) == digest(Hp, ap), f"pinned and pageable differ bitwise; {note}"


# ---------------------------------------------------------------------------------------------------------------------
# 7. a zero column in a late chunk
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", F.NAN_FAMILIES)
def test_zero_column_in_a_late_chunk(D, h, oracle, coracle, family):
    m, n = 2048, 1024
    ref = Ref(coracle, oracle, family, m, n)
    for cu in (1, 3):
        with host_options(h, host_cu_streams=cu, **DEADLINE) as o:
            bounds, join = plan(D, o, m, n, 0)
            with np.errstate(all="ignore"):
                H, a, _, note = host_qr(D, h, ref.A)
        note += "; " + windowed(bounds, join)
        assert F.zero_column(family, n) >= bounds[2], note
        hold(f"deadline cu{cu}", ref, H, a, note)


# ---------------------------------------------------------------------------------------------------------------------
# 8. the Python layer on a pinned buffer
# ---------------------------------------------------------------------------------------------------------------------
def test_python_layer_on_a_pinned_buffer(D, h):
    m, n = 2048, 1024
    A0 = F.make("graded6", m, n)
    b0 = F.rhs(m)
    with host_options(h, **DEADLINE) as o:
        _, view = pinned(A0)
        An = view.numpy()
        assert An.flags.f_contiguous and not An.flags.owndata
        st = D.qr_(An, handle=h)
        b = b0.copy()
        x = D.ldiv(st, b)
        H, a, _, _ = host_qr(D, h, A0)
        x2 = host_ldiv(D, h, H, a, b0)
    assert np.array_equal(b, b0), "ldiv wrote to b"
    assert digest(An, st.α) == digest(H, a), "qr_ on a pinned numpy view differs bitwise from dhqr_qr_host_f64"
    assert digest(x) == digest(x2), "ldiv differs bitwise from dhqr_ldiv_host_f64"
