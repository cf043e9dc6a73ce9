"""Every entry point returns the same bits whatever its handle did before (run with -m gpu on an H100).

A handle lives for a whole program (the Python default_handle, the Julia shim's per-device handle, a StreamingLeastSquares that
appends and solves for as long as rows arrive), and every entry point shares its state: the workspace sets, the V buffers, the
wide chain's control words, the exchange cells with their launch-tag counters (ll_epoch for k_panel and k_tp_panel, bs_epoch for
both wavefront substitutions, uw_epoch for the nb = 1 wave).  Workspace is zero-filled only when it grows, so a fresh handle
hands every kernel zeros while a used one hands it whatever the last call left.  Every result of the library is bitwise
deterministic (fixed-order split-K sums, split counts set by the shape and the SM count), so the check is exact: after any
history, a call gives the bits of the same call on a fresh handle.

CASES is the catalogue: one or more cases per C-ABI function that enqueues work, each a function of (handle, stream) whose
outputs are everything the call writes.  test_catalogue_covers_the_header (no GPU) holds the catalogue to include/dhqr.h.  The
reference bits come from a fresh handle per case; the histories are:
  grown by others     one call per workspace owner at a larger shape, so every buffer grows and holds non-zero data
  pair walk           every case directly after every case (an Euler circuit of the complete digraph with loops: N^2 + 1 runs)
  refusal             a qr_ whose 128-column panel the wide chain refused and the 32-column chain redid
  argument errors     one rejected call per entry point: no launch, no trace
  options             each writable option set, one qr_ and one solve (the host pair for the host_* keys), the option restored
  random orders       the whole catalogue in two seeded orders on one handle
  two handles         two handles on their own non-blocking streams, fed alternately from one thread without synchronising
  epoch wraps         the tag counters moved next to their resets (option "epoch_near_wrap"), calls before, across and after
"""
import ctypes as C
import hashlib
import os
import re
import time

import numpy as np
import pytest
import torch

import dhqr_b200 as D
import matrix_families as F
from ext_rule import options

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
M, N = 1000, 300           # catalogue shape: nb = 1 goes through k_unblocked_wave (m <= 8192), two wide panels + a narrow one
RANK = 250                 # rank of the pivoted cases' input
MT, NT = 8200, 64          # nb = 1 above the wave's 8192 rows: one k_apply1_tma launch per column
KA = 500                   # rows appended
MH, NH = 1536, 1536        # host entry: upload chunks [0, 384, 768, 1280, 1536], the last two joining after a catch-up
NBR = 128                  # columns of the block-reflector hook


def P(t):
    return C.c_void_p(t.data_ptr())


def SP(s):
    return C.c_void_p(s.cuda_stream)


def call(name, *args):
    D._lib.call(name, *args)


def up(x):
    """Host array -> device, on the current stream: a 1-D tensor, or a column-major (m, n) one with lda = m."""
    t = torch.from_numpy(np.ascontiguousarray(x) if x.ndim == 1 else np.asfortranarray(x))
    if x.ndim == 1:
        return t.to(DEV)
    out = D.colmajor_empty(x.shape[0], x.shape[1], DEV, dtype=t.dtype)
    out.copy_(t)
    return out


def zeros(n, dtype=torch.float64):
    return torch.zeros(n, dtype=dtype, device=DEV)


def nrhs_of(b):
    return 1 if b.ndim == 1 else b.shape[1]


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue: name -> (C functions it calls, fn(h, s, X) -> {output: tensor or array}).  X holds the host inputs.
# ---------------------------------------------------------------------------------------------------------------------
CASES = {}


def case(name, *fns):
    def reg(f):
        CASES[name] = (fns, f)
        return f
    return reg


def _qr(h, s, A0, nb=0):
    m, n = A0.shape
    A, al = up(A0), zeros(n)
    call("dhqr_qr_f64", h.raw, m, n, 0, n, P(A), m, P(al), nb, SP(s))
    return {"A": A, "alpha": al}


case("qr_f64", "dhqr_qr_f64")(lambda h, s, X: _qr(h, s, X["A"]))
case("qr_f64_nb64", "dhqr_qr_f64")(lambda h, s, X: _qr(h, s, X["A"], 64))
case("qr_f64_nb1_wave", "dhqr_qr_f64")(lambda h, s, X: _qr(h, s, X["A"], 1))
case("qr_f64_nb1_tall", "dhqr_qr_f64")(lambda h, s, X: _qr(h, s, X["At"], 1))


@case("qr_f64_wide_panel0", "dhqr_qr_f64")
def _qr_wide0(h, s, X):
    with options(h, wide_panel=0):          # every panel through k_panel: the tag-heavy path
        return _qr(h, s, X["A"])


def _sweep(h, s, fn, A0, b0):               # apply_qt / apply_q: (h, m, n, col0, nl, A, lda, b, ldb, nrhs, s)
    A, b = up(A0), up(b0)
    call(fn, h.raw, M, N, 0, N, P(A), M, P(b), M, nrhs_of(b0), SP(s))
    return {"b": b}


def _tri(h, s, fn, A0, al0, b0):            # backsolve / solve: (h, m, n, col0, nl, A, lda, alpha, b, ldb, nrhs, s)
    A, al, b = up(A0), up(al0), up(b0)
    call(fn, h.raw, M, N, 0, N, P(A), M, P(al), P(b), M, nrhs_of(b0), SP(s))
    return {"b": b}


for _r in (1, 3):
    case(f"apply_qt_f64_r{_r}", "dhqr_apply_qt_f64")(lambda h, s, X, r=_r: _sweep(h, s, "dhqr_apply_qt_f64", X["H"], X[f"b{r}"]))
    case(f"apply_q_f64_r{_r}", "dhqr_apply_q_f64")(lambda h, s, X, r=_r: _sweep(h, s, "dhqr_apply_q_f64", X["H"], X[f"b{r}"]))
    case(f"backsolve_f64_r{_r}", "dhqr_backsolve_f64")(
        lambda h, s, X, r=_r: _tri(h, s, "dhqr_backsolve_f64", X["H"], X["alpha"], X[f"b{r}"]))
    case(f"solve_f64_r{_r}", "dhqr_solve_f64")(lambda h, s, X, r=_r: _tri(h, s, "dhqr_solve_f64", X["H"], X["alpha"], X[f"b{r}"]))
    case(f"apply_qt_c64_r{_r}", "dhqr_apply_qt_c64")(lambda h, s, X, r=_r: _sweep(h, s, "dhqr_apply_qt_c64", X["Hc"], X[f"c{r}"]))
    case(f"backsolve_c64_r{_r}", "dhqr_backsolve_c64")(
        lambda h, s, X, r=_r: _tri(h, s, "dhqr_backsolve_c64", X["Hc"], X["alphac"], X[f"c{r}"]))
    case(f"solve_c64_r{_r}", "dhqr_solve_c64")(lambda h, s, X, r=_r: _tri(h, s, "dhqr_solve_c64", X["Hc"], X["alphac"], X[f"c{r}"]))


@case("qr_c64", "dhqr_qr_c64")
def _qr_c64(h, s, X):
    A, al = up(X["Ac"]), zeros(N, torch.complex128)
    call("dhqr_qr_c64", h.raw, M, N, 0, N, P(A), M, P(al), SP(s))
    return {"A": A, "alpha": al}


def _form_q(h, s, fn, A0):
    A = up(A0)
    Q = D.colmajor_empty(M, N, DEV, dtype=A.dtype)
    call(fn, h.raw, M, N, P(A), M, P(Q), M, SP(s))
    return {"Q": Q}


case("form_q_f64", "dhqr_form_q_f64")(lambda h, s, X: _form_q(h, s, "dhqr_form_q_f64", X["H"]))
case("form_q_c64", "dhqr_form_q_c64")(lambda h, s, X: _form_q(h, s, "dhqr_form_q_c64", X["Hc"]))


def _adj(h, s, fn, A0, al0, b0):            # forwardsolve / solve_adj: (h, m, n, A, lda, alpha, b, ldb, nrhs, s)
    A, al, b = up(A0), up(al0), up(b0)
    call(fn, h.raw, M, N, P(A), M, P(al), P(b), M, nrhs_of(b0), SP(s))
    return {"b": b}


case("forwardsolve_f64_r3", "dhqr_forwardsolve_f64")(lambda h, s, X: _adj(h, s, "dhqr_forwardsolve_f64", X["H"], X["alpha"], X["b3"]))
case("forwardsolve_c64_r3", "dhqr_forwardsolve_c64")(lambda h, s, X: _adj(h, s, "dhqr_forwardsolve_c64", X["Hc"], X["alphac"], X["c3"]))
case("solve_adj_f64_r1", "dhqr_solve_adj_f64")(lambda h, s, X: _adj(h, s, "dhqr_solve_adj_f64", X["H"], X["alpha"], X["b1"]))
case("solve_adj_c64_r1", "dhqr_solve_adj_c64")(lambda h, s, X: _adj(h, s, "dhqr_solve_adj_c64", X["Hc"], X["alphac"], X["c1"]))


for _t, _cd in (("f64", torch.float64), ("c64", torch.complex128)):
    _p = "" if _t == "f64" else "c"     # X keys of the complex twins

    @case(f"qrcp_{_t}", f"dhqr_qrcp_{_t}")
    def _qrcp(h, s, X, t=_t, p=_p, cd=_cd):
        A, al, jp = up(X[p + "Ar"]), zeros(N, cd), zeros(N, torch.int64)
        call(f"dhqr_qrcp_{t}", h.raw, M, N, P(A), M, P(al), P(jp), SP(s))
        return {"A": A, "alpha": al, "jpvt": jp}

    @case(f"solve_qrcp_{_t}_r3", f"dhqr_solve_qrcp_{_t}")
    def _solve_qrcp(h, s, X, t=_t, p=_p):
        A, al, jp, b = up(X[p + "HP"]), up(X[p + "alphaP"]), up(X[p + "jpvt"]), up(X[p + "br3"])
        call(f"dhqr_solve_qrcp_{t}", h.raw, M, N, RANK, P(A), M, P(al), P(jp), P(b), M, 3, SP(s))
        return {"b": b}

    @case(f"cod_{_t}", f"dhqr_cod_{_t}")
    def _cod(h, s, X, t=_t, p=_p, cd=_cd):
        A, al = up(X[p + "HP"]), up(X[p + "alphaP"])
        Fm, g = D.colmajor_empty(N, RANK, DEV, dtype=cd), zeros(RANK, cd)
        call(f"dhqr_cod_{t}", h.raw, M, N, RANK, P(A), M, P(al), P(Fm), N, P(g), SP(s))
        return {"F": Fm, "gamma": g}

    @case(f"solve_cod_{_t}_r3", f"dhqr_solve_cod_{_t}")
    def _solve_cod(h, s, X, t=_t, p=_p):
        A, jp, Fm, g, b = up(X[p + "HP"]), up(X[p + "jpvt"]), up(X[p + "F"]), up(X[p + "gamma"]), up(X[p + "br3"])
        call(f"dhqr_solve_cod_{t}", h.raw, M, N, RANK, P(A), M, P(jp), P(Fm), N, P(g), P(b), M, 3, SP(s))
        return {"b": b}


@case("qr_append", "dhqr_qr_append_f64")
def _append(h, s, X):
    R, al, B, vt = up(X["H"]), up(X["alpha"]), up(X["B"]), zeros(N)
    call("dhqr_qr_append_f64", h.raw, N, KA, P(R), M, P(al), P(B), KA, P(vt), SP(s))
    return {"R": R, "alpha": al, "B": B, "vtop": vt}


def _apply_append(h, s, fn, X):
    B, vt, c, e = up(X["V2"]), up(X["vtop"]), up(X["ca"]), up(X["ea"])
    call(fn, h.raw, N, KA, P(B), KA, P(vt), P(c), N, P(e), KA, 3, SP(s))
    return {"c": c, "e": e}


case("apply_qt_append_r3", "dhqr_apply_qt_append_f64")(lambda h, s, X: _apply_append(h, s, "dhqr_apply_qt_append_f64", X))
case("apply_q_append_r3", "dhqr_apply_q_append_f64")(lambda h, s, X: _apply_append(h, s, "dhqr_apply_q_append_f64", X))


@case("streaming_lstsq", "dhqr_qr_append_f64", "dhqr_apply_qt_append_f64", "dhqr_backsolve_f64")
def _streaming(h, s, X):
    ls = D.StreamingLeastSquares(N, nrhs=2, device=0, handle=h)         # R = 0, then three blocks
    for r0 in range(0, X["As"].shape[0], 400):
        ls.add(torch.from_numpy(X["As"][r0:r0 + 400]).to(DEV), torch.from_numpy(X["bs"][r0:r0 + 400]).to(DEV))
    return {"R": ls.A, "alpha": ls.α, "c": ls.c, "ss": ls._ss, "x": ls.solve()}


@case("host_qr_ldiv", "dhqr_qr_host_f64", "dhqr_ldiv_host_f64")
def _host(h, s, X):
    hA = torch.empty((NH, MH), dtype=torch.float64, pin_memory=True).numpy().T     # Fortran-ordered, pinned
    hA[:] = X["Ah"]
    st = D.qr_(hA, handle=h)
    x = D.ldiv(st, X["bh"])
    return {"A": hA, "alpha": st.α, "x": x}


def _pdot(h, s, fn, a0, b0):
    a, b, out = up(a0), up(b0), zeros(1, torch.from_numpy(a0[:1]).dtype)
    call(fn, h.raw, P(a), P(b), 3, M - 3, P(out), SP(s))
    return {"dot": out}


case("partialdot_f64", "dhqr_partialdot_f64")(lambda h, s, X: _pdot(h, s, "dhqr_partialdot_f64", X["b1"], X["b3"][:, 1]))
case("partialdot_c64", "dhqr_partialdot_c64")(lambda h, s, X: _pdot(h, s, "dhqr_partialdot_c64", X["c1"], X["c3"][:, 1]))


@case("fill_uniform", "dhqr_fill_uniform_f64")
def _fill(h, s, X):
    A = D.colmajor_empty(M, N, DEV)
    call("dhqr_fill_uniform_f64", h.raw, 7, 5, 11, M, N, P(A), M, SP(s))
    return {"A": A}


@case("k_block_reflector", "dhqr_k_block_reflector_f64")
def _kbr(h, s, X):
    V, Cm, L = up(X["V"]), up(X["Cb"]), zeros(NBR * NBR)
    call("dhqr_k_block_reflector_f64", h.raw, M, NBR, P(V), M, 0, 200, P(Cm), M, P(L), SP(s))
    return {"C": Cm, "linv": L}


@case("k_panel", "dhqr_k_panel_f64")
def _kpanel(h, s, X):
    Pm, al = up(X["A"][:, :32]), zeros(32)
    call("dhqr_k_panel_f64", h.raw, M, 32, P(Pm), M, P(al), SP(s))
    return {"P": Pm, "alpha": al}


@case("k_wide_panel", "dhqr_k_wide_panel_f64")
def _kwide(h, s, X):
    Pm, al, refused = up(X["A"][:, :128]), zeros(128), C.c_int(-1)
    call("dhqr_k_wide_panel_f64", h.raw, M, P(Pm), M, P(al), C.byref(refused), SP(s))
    return {"P": Pm, "alpha": al, "refused": np.array([refused.value])}


# functions of include/dhqr.h that enqueue no work of their own, or whose results are not results
EXCLUDED = {
    "dhqr_version": "library constant",
    "dhqr_last_error": "host-side error text",
    "dhqr_create": "creates the handle every case runs on",
    "dhqr_create_dist": "multi-rank handles: their contract is held by the loopback harness",
    "dhqr_destroy": "ends the handle's history",
    "dhqr_nccl_unique_id": "host-side NCCL id, no device work",
    "dhqr_set_option": "part of the histories (options set and restored, epoch_near_wrap), not a result",
    "dhqr_get_option": "reads options and counters, writes nothing",
    "dhqr_launch_count": "read-only counter",
    "dhqr_profile_reset": "clears host-side profile accumulators",
    "dhqr_profile_get": "reads profile accumulators",
    "dhqr_plan_host_upload": "pure host logic, needs no device",
    "dhqr_debug_copy_f64": "copies internal workspace out: debugging, not a result",
}


def _header_functions():
    src = open(os.path.join(ROOT, "include", "dhqr.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(dhqr_[a-z0-9_]+)\s*\(", src))


def test_catalogue_covers_the_header():
    """Every function of include/dhqr.h is in the catalogue or excluded with a reason, and neither list names one it lacks."""
    declared = _header_functions()
    covered = {f for fns, _ in CASES.values() for f in fns}
    assert not covered & set(EXCLUDED), f"both in the catalogue and excluded: {sorted(covered & set(EXCLUDED))}"
    missing = declared - covered - set(EXCLUDED)
    assert not missing, f"entry points with no history case and no reason to be left out: {sorted(missing)}"
    unknown = (covered | set(EXCLUDED)) - declared
    assert not unknown, f"not declared in include/dhqr.h: {sorted(unknown)}"


# ---------------------------------------------------------------------------------------------------------------------
# running and comparing
# ---------------------------------------------------------------------------------------------------------------------
def run(name, h, s, X):
    with torch.cuda.stream(s):
        return CASES[name][1](h, s, X)


def digests(outs, s):
    s.synchronize()
    return {k: hashlib.sha256(np.ascontiguousarray(v.cpu().numpy() if torch.is_tensor(v) else v).tobytes()).hexdigest()
            for k, v in outs.items()}


def differing(name, got, ref):
    return [f"{name}.{k}" for k in ref[name] if got.get(k) != ref[name][k]]


def check_all(h, s, X, ref, prelude, names=None):
    bad = []
    for name in names or CASES:
        bad += differing(name, digests(run(name, h, s, X), s), ref)
    assert not bad, f"after {prelude}: {bad} differ from the bits of a fresh handle"


class Fresh:
    """A handle on its own non-blocking stream, destroyed on exit."""

    def __enter__(self):
        self.h, self.s = D.Handle(0), torch.cuda.Stream()
        return self.h, self.s

    def __exit__(self, *exc):
        self.s.synchronize()
        self.h.close()


@pytest.fixture(scope="module")
def X():
    """Host inputs.  The factorisations the solve cases read are made by the catalogue's own cases, on a scratch handle."""
    assert torch.cuda.is_available()
    x = {"A": F.make("normal", M, N), "At": F.make("normal", MT, NT), "Ac": F.make_complex("centered", M, N),
         "b1": F.rhs(M, 1), "b3": F.rhs(M, 3), "c1": F.rhs(M, 1, cplx=True), "c3": F.rhs(M, 3, cplx=True),
         "B": F.make("normal", KA, N), "ca": F.rhs(N, 3, seed=1), "ea": F.rhs(KA, 3, seed=2),
         "As": F.make("normal", 1200, N, seed=3), "bs": F.rhs(1200, 2, seed=3),
         "Ah": F.make("normal", MH, NH), "bh": F.rhs(MH, 1, seed=4), "Cb": F.make("normal", M, 200, seed=5),
         "br3": F.rhs(M, 3, seed=6), "cbr3": F.rhs(M, 3, seed=6, cplx=True)}
    x["Ar"] = np.asfortranarray(F.make("normal", M, RANK) @ F.make("normal", N, RANK).T)
    x["cAr"] = np.asfortranarray(F.make_complex("normal", M, RANK) @ F.make_complex("normal", N, RANK).T)

    def host(outs):
        torch.cuda.synchronize()
        return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in outs.items()}

    with Fresh() as (h, s):
        o = host(run("qr_f64", h, s, x))
        x["H"], x["alpha"] = o["A"], o["alpha"]
        x["V"] = np.asfortranarray(np.tril(x["H"][:, :NBR]))
        o = host(run("qr_c64", h, s, x))
        x["Hc"], x["alphac"] = o["A"], o["alpha"]
        for p in ("", "c"):
            t = "f64" if p == "" else "c64"
            o = host(run(f"qrcp_{t}", h, s, x))
            x[p + "HP"], x[p + "alphaP"], x[p + "jpvt"] = o["A"], o["alpha"], o["jpvt"]
            o = host(run(f"cod_{t}", h, s, x))
            x[p + "F"], x[p + "gamma"] = o["F"], o["gamma"]
        o = host(run("qr_append", h, s, x))
        x["V2"], x["vtop"] = o["B"], o["vtop"]
    return x


@pytest.fixture(scope="module")
def REF(X):
    """Bits of every case on a fresh handle, and a check that each case calls the C functions the catalogue says it does."""
    ref, seen = {}, {}
    real = D._lib.call

    def spy(name, *args):
        seen.setdefault(current, set()).add(name)
        return real(name, *args)

    D._lib.call = spy
    try:
        for current in CASES:
            with Fresh() as (h, s):
                ref[current] = digests(run(current, h, s, X), s)
    finally:
        D._lib.call = real
    for name, (fns, _) in CASES.items():
        assert set(fns) <= seen.get(name, set()), f"{name} does not call {sorted(set(fns) - seen.get(name, set()))}"
    return ref


# ---------------------------------------------------------------------------------------------------------------------
# histories
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fresh_handles_agree(X, REF):
    """A second fresh handle gives the reference bits (they are a fixed point, not one sample), and the wide-chain hook
    accepts the catalogue's well-conditioned panel."""
    with Fresh() as (h, s):
        check_all(h, s, X, REF, "nothing (a second fresh handle per case)", names=["qr_f64", "k_wide_panel", "solve_f64_r1"])
    with Fresh() as (h, s):
        assert run("k_wide_panel", h, s, X)["refused"][0] == 0


def grow(h, s):
    """One call per workspace owner at a larger shape than any case's, leaving non-zero data in every buffer."""
    with torch.cuda.stream(s):
        _qr(h, s, F.make("normal", 8192, 1024, seed=9))                       # vpk2 / vpkb / ws[0..2], linv_all, gram_all, wbuf
        _qr(h, s, F.make("normal", 4096, 1000, seed=9), 64)                    # k_panel cells over many CTAs, narrow chain
        hA = torch.empty((2048, 3000), dtype=torch.float64, pin_memory=True).numpy().T
        hA[:] = F.make("normal", 3000, 2048, seed=9)                          # chunks join at steps 0, 0, 1, 2, 3: catch-up sets 3-5
        D.qr_(hA, handle=h)
        nb = 2048                                                              # bs_cells and xbuf: 64 strips, 65 right-hand sides
        A, al, b = up(F.make("normal", nb, nb, seed=9)), torch.full((nb,), 64.0, dtype=torch.float64, device=DEV), up(F.rhs(nb, 65, seed=9))
        call("dhqr_backsolve_f64", h.raw, nb, nb, 0, nb, P(A), nb, P(al), P(b), nb, 65, SP(s))
        call("dhqr_forwardsolve_f64", h.raw, nb, nb, P(A), nb, P(al), P(b), nb, 65, SP(s))
        A, al, jp = up(F.make("normal", 2048, 1024, seed=9)), zeros(1024), zeros(1024, torch.int64)
        call("dhqr_qrcp_f64", h.raw, 2048, 1024, P(A), 2048, P(al), P(jp), SP(s))   # qp_buf, qp_flag
        Ac, alc, jpc = up(F.make_complex("normal", 2048, 512, seed=9)), zeros(512, torch.complex128), zeros(512, torch.int64)
        call("dhqr_qrcp_c64", h.raw, 2048, 512, P(Ac), 2048, P(alc), P(jpc), SP(s))
        Ac = up(F.make_complex("normal", 2048, 512, seed=9))
        call("dhqr_qr_c64", h.raw, 2048, 512, 0, 512, P(Ac), 2048, P(alc), SP(s))
        k, n = h.get_option("append_max_rows") // 8, 512                       # the append near its slab capacity / 8
        R, al, B, vt = up(np.triu(F.make("normal", n, n, seed=9))), zeros(n), up(F.make("normal", k, n, seed=9)), zeros(n)
        call("dhqr_qr_append_f64", h.raw, n, k, P(R), n, P(al), P(B), k, P(vt), SP(s))
        _qr(h, s, F.make("normal", 4096, 1024, seed=9), 1)                     # uw_flags: the nb = 1 wave at n = 1024
        A = _qr(h, s, F.make("normal", 60000, 128, seed=9))["A"]               # qt_part / qt_T: the Q'b sweep over 60000 rows
        b = up(F.rhs(60000, 1, seed=9))
        call("dhqr_apply_qt_f64", h.raw, 60000, 128, 0, 128, P(A), 60000, P(b), 60000, 1, SP(s))
    s.synchronize()


@pytest.mark.gpu
def test_after_larger_calls_of_every_workspace_owner(X, REF):
    with Fresh() as (h, s):
        grow(h, s)
        check_all(h, s, X, REF, "calls at larger shapes that grew every workspace buffer (8192 x 1024 qr_, host entry with 3 "
                                "catch-ups, nrhs 65 substitutions, qrcp, the append at append_max_rows / 8, the nb = 1 wave, the "
                                "Q'b sweep at 60000 rows)")


def euler_walk(names):
    """A sequence in which every ordered pair (a, b), a == b included, appears exactly once as neighbours (Hierholzer)."""
    left = {i: list(range(len(names))) for i in range(len(names))}
    stack, path = [0], []
    while stack:
        v = stack[-1]
        if left[v]:
            stack.append(left[v].pop())
        else:
            path.append(stack.pop())
    return [names[i] for i in reversed(path)]


def test_euler_walk_covers_every_pair():
    names = list(CASES)
    walk = euler_walk(names)
    pairs = list(zip(walk, walk[1:]))
    assert len(pairs) == len(names) ** 2 and set(pairs) == {(a, b) for a in names for b in names}


@pytest.mark.gpu
def test_every_case_after_every_case(X, REF):
    walk = euler_walk(list(CASES))
    bad = []
    t0 = time.perf_counter()
    with Fresh() as (h, s):
        for i, name in enumerate(walk):
            got = digests(run(name, h, s, X), s)
            bad += [f"{d} after {walk[i - 1] if i else 'nothing'} (step {i})" for d in differing(name, got, REF)]
    print(f"pair walk: {len(walk)} runs in {time.perf_counter() - t0:.1f} s")
    assert not bad, f"{len(bad)} results differ from the bits of a fresh handle: {bad[:20]}"


@pytest.mark.gpu
def test_after_a_refused_wide_panel(X, REF):
    A0 = F.make("normal", 3000, 640, seed=8)
    A0[:, 200] = A0[:, 150] + 1e-11 * F.rhs(3000, 1, seed=8)             # the second outer panel nearly rank deficient
    with Fresh() as (h, s):
        r0 = h.get_option("wide_redone")
        with torch.cuda.stream(s):
            _qr(h, s, A0)
        s.synchronize()
        assert h.get_option("wide_redone") == r0 + 1
        check_all(h, s, X, REF, "a qr_ whose second wide panel was refused and redone by the 32-column chain")


def bad_args(name, h):
    """Every size -1, every pointer null: an argument error on a valid handle."""
    out = []
    for i, t in enumerate(D._lib.SIGNATURES[name]):
        if i == 0:
            out.append(h.raw)
        elif t in (C.c_int64, C.c_int):
            out.append(-1)
        elif t is C.c_uint64:
            out.append(0)
        else:
            out.append(None)
    return out


@pytest.mark.gpu
def test_after_argument_errors(X, REF):
    lib = D._lib.load()
    fns = sorted({f for fns, _ in CASES.values() for f in fns})
    with Fresh() as (h, s):
        for name in CASES:                          # the buffers exist, so an error cannot hide behind a first allocation
            run(name, h, s, X)
        s.synchronize()
        n0 = h.launch_count()
        for name in fns:
            rc = getattr(lib, name)(*bad_args(name, h))
            assert rc < 0, f"{name} with every size -1 and every pointer null returned {rc}"
        assert h.launch_count() == n0, "a rejected call launched a kernel"
        check_all(h, s, X, REF, f"one rejected call of each of {len(fns)} entry points")


# writable option -> (a non-default value, its default)
OPTION_CHANGES = {"nb": (64, 128), "lookahead": (0, 1), "wide_panel": (0, 1), "panel_fast": (0, 1), "panel_ctas": (48, 0),
                  "cvy_persist": (2, 4), "qt_vec": (0, 1), "bs_wave": (0, 1), "unblocked_wave": (0, 1), "fuse_house": (0, 1),
                  "wide_kappa": (100, 1000), "host_chunk": (256, 512), "host_first": (512, 0), "host_h2d_gbs": (25, 50),
                  "host_tflops": (40, 27), "host_chain_us": (200, 300), "host_cu_streams": (2, 3), "host_trace": (1, 0),
                  "profile": (1, 0), "sync": (1, 0), "panel_trace": (1, 0), "la_trace": (1, 0), "wide_trace": (1, 0),
                  "chain_wait_trace": (1, 0)}


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(OPTION_CHANGES))
def test_after_an_option_set_and_restored(X, REF, key):
    val, default = OPTION_CHANGES[key]
    pair = ("host_qr_ldiv",) if key.startswith("host_") else ("qr_f64", "solve_f64_r1")
    with Fresh() as (h, s):
        h.set_option(key, val)
        for name in pair:
            run(name, h, s, X)
        s.synchronize()
        h.set_option(key, default)                   # no profile_reset: brackets left pending by "profile" stay on the handle
        check_all(h, s, X, REF, f"option {key} = {val}, {' + '.join(pair)}, option back to {default}")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", (1, 2))
def test_catalogue_in_a_random_order(X, REF, seed):
    order = [list(CASES)[i] for i in np.random.default_rng(seed).permutation(len(CASES))]
    bad = []
    with Fresh() as (h, s):
        for i, name in enumerate(order):
            got = digests(run(name, h, s, X), s)
            bad += [f"{d} after {order[max(0, i - 3):i]}" for d in differing(name, got, REF)]
    assert not bad, f"seed {seed}: {bad}"


@pytest.mark.gpu
def test_two_handles_on_one_device(X, REF):
    """Handles A and B on their own non-blocking streams, fed alternately from this thread with no synchronisation between them:
    A runs the catalogue in order, B in reverse, and both must give the fresh bits.  Only the host entry points, the wide-chain
    hook and a qr_ whose panel went through the wide chain synchronise, each its own stream (include/dhqr.h).

    Kernels that wait on a word another CTA writes (CTAs of one launch may then share the device with the other handle's work):
      k_panel, k_tp_panel, k_unblocked_wave   cooperative launches: the driver makes every CTA resident before any starts
      k_gemm_cvy_p                            waits on mbarriers of its own 2-CTA cluster, which the hardware co-schedules;
                                              its read of the wide chain's fail_step does not wait
      k_forwardsolve_wave                     CTA k waits on the x cells of CTAs 0 .. k - 1 only
      k_backsolve_wave                        CTA i owns block nbk - 1 - i and waits on blocks above it, i.e. on CTAs 0 .. i - 1
                                              only; the update-only CTAs of the rows above a rank's columns come after all of them
    The wide chain (dhqr_wide.cuh) has no spinning CTAs, and the last-CTA tickets of k_qt_dot and the pivoted path's reductions
    never wait.  CTAs are dispatched in index order, so when only some CTAs of a wave are resident, the resident ones include
    the lowest-numbered waiting CTA's every predecessor: CTA 0 needs nothing, and each CTA that finishes frees a slot for the
    next.  Neither wave can stall on CTAs that are not yet resident, whatever the other handle keeps on the device."""
    names = list(CASES)
    with Fresh() as (ha, sa), Fresh() as (hb, sb):
        outs_a, outs_b = {}, {}
        for i in range(len(names)):
            outs_a[names[i]] = run(names[i], ha, sa, X)
            outs_b[names[-1 - i]] = run(names[-1 - i], hb, sb, X)
        bad = []
        for tag, outs, s in (("A", outs_a, sa), ("B", outs_b, sb)):
            for name, o in outs.items():
                bad += [f"handle {tag}: {d}" for d in differing(name, digests(o, s), REF)]
    assert not bad, f"two handles working at once on one device: {bad}"


# the cases that cross each tag reset, and the counter they advance: 0 = ll_epoch, 1 = bs_epoch, 2 = uw_epoch
EPOCH_CASES = {"qr_f64_wide_panel0": 0, "qr_append": 0, "backsolve_f64_r3": 1, "forwardsolve_f64_r3": 1, "qr_f64_nb1_wave": 2}
LL_MAX, WAVE_MAX = 0xF0000000, 0xFFFFFFF0          # reset thresholds (dhqr_api.cu); a k_panel / k_tp_panel launch takes 40 tags
NEAR = {0: LL_MAX - 2 * 40 + 1, 1: WAVE_MAX - 1, 2: WAVE_MAX - 1}


def epochs(h, s):
    out = torch.zeros(3, dtype=torch.float64, device=DEV)
    call("dhqr_debug_copy_f64", h.raw, b"epochs", P(out), 3, SP(s))
    return [int(v) for v in out.cpu().tolist()]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EPOCH_CASES))
def test_across_every_epoch_reset(X, REF, name):
    """The tag counters two launches below their resets (option "epoch_near_wrap"), then the case three times: launches before
    the reset use the top tags, the reset clears the cells, the launches after it start over at tag 1.  Every run must give
    the fresh bits, and the counters read back must show that the reset ran."""
    idx = EPOCH_CASES[name]
    with Fresh() as (h, s):
        assert not differing(name, digests(run(name, h, s, X), s), REF)       # buffers allocated: the hook now sticks
        h.set_option("epoch_near_wrap", 1)
        seen = [epochs(h, s)]
        assert seen[0][idx] == NEAR[idx], seen
        bad = []
        for i in range(3):
            bad += [f"{d} (run {i} after epoch_near_wrap; counters {seen[-1]})" for d in differing(name, digests(run(name, h, s, X), s), REF)]
            seen.append(epochs(h, s))
        assert not bad, bad
        drops = [i for i in range(3) if seen[i + 1][idx] < seen[i][idx]]
        assert drops, f"{name}: counter {idx} never reset: {seen}"
        assert seen[drops[0]][idx] >= NEAR[idx], f"{name}: the reset came before the top tags were used: {seen}"
