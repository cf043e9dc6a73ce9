"""Option "profile": every kernel launch is bracketed and timed in a class.  For each entry point, the per-class counts of one call
add up to the launches it made (dhqr_launch_count), and every class has a name, so the profile accounts for a whole call."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def p(t):
    return C.c_void_p(t.data_ptr())


def f64(D, h, m, n, seed):
    A = D.colmajor_empty(m, n, DEV)
    D.fill_uniform_(A, seed, handle=h)
    return A


def c64(m, n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    re = torch.rand((n, m), generator=g, device=DEV, dtype=torch.float64) - 0.5
    im = torch.rand((n, m), generator=g, device=DEV, dtype=torch.float64) - 0.5
    return torch.complex(re, im).t()                                   # column-major, lda = m


def factored(D, h, m, n, seed=1):
    A, al = f64(D, h, m, n, seed), torch.zeros(n, dtype=torch.float64, device=DEV)
    D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, p(A), m, p(al), 0, None)
    return A, al


def factored_c64(D, h, m, n, seed=1):
    A, al = c64(m, n, seed), torch.zeros(n, dtype=torch.complex128, device=DEV)
    D._lib.call("dhqr_qr_c64", h.raw, m, n, 0, n, p(A), m, p(al), None)
    return A, al


# Each case prepares its inputs on the handle and returns the one call to account for.
def qr_case(m, n, nb, **opts):
    def make(D, h):
        for k, v in opts.items():
            h.set_option(k, v)
        A, al = f64(D, h, m, n, 3), torch.zeros(n, dtype=torch.float64, device=DEV)
        return lambda: D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, p(A), m, p(al), nb, None)
    return make


def refused_pair(D, h):
    # test_gpu_wide.py::test_restart_after_a_refused_panel: the second panel of the first pair is refused; the restart re-packs
    # the first panel (k_pack) and applies it right of the pair before it redoes the second
    m, n = 3000, 640
    A = f64(D, h, m, n, 12)
    A[:, 200] = A[:, 150] + 1e-11 * f64(D, h, m, 1, 13)[:, 0]
    al = torch.zeros(n, dtype=torch.float64, device=DEV)
    return lambda: D._lib.call("dhqr_qr_f64", h.raw, m, n, 0, n, p(A), m, p(al), 0, None)


def apply_case(fn, nrhs):
    def make(D, h):
        m, n = 1024, 300
        A, _ = factored(D, h, m, n)
        b = f64(D, h, m, nrhs, 5)
        return lambda: D._lib.call(fn, h.raw, m, n, 0, n, p(A), m, p(b), m, nrhs, None)
    return make


def backsolve_case(wave):
    def make(D, h):
        h.set_option("bs_wave", wave)
        m, n, nrhs = 1024, 300, 2
        A, al = factored(D, h, m, n)
        b = f64(D, h, m, nrhs, 5)
        return lambda: D._lib.call("dhqr_backsolve_f64", h.raw, m, n, 0, n, p(A), m, p(al), p(b), m, nrhs, None)
    return make


def adj_case(fn, cplx):
    def make(D, h):
        m, n, nrhs = 1024, 300, 2
        A, al = factored_c64(D, h, m, n) if cplx else factored(D, h, m, n)
        b = c64(m, nrhs, 5) if cplx else f64(D, h, m, nrhs, 5)
        return lambda: D._lib.call(fn, h.raw, m, n, p(A), m, p(al), p(b), m, nrhs, None)
    return make


def form_q_case(cplx):
    def make(D, h):
        m, n = 1024, 300
        A, _ = factored_c64(D, h, m, n) if cplx else factored(D, h, m, n)
        Q = torch.empty_like(A.t()).t()
        return lambda: D._lib.call("dhqr_form_q_c64" if cplx else "dhqr_form_q_f64", h.raw, m, n, p(A), m, p(Q), m, None)
    return make


def qr_c64(D, h):
    m, n = 1024, 300
    A, al = c64(m, n, 3), torch.zeros(n, dtype=torch.complex128, device=DEV)
    return lambda: D._lib.call("dhqr_qr_c64", h.raw, m, n, 0, n, p(A), m, p(al), None)


def apply_qt_c64(D, h):
    m, n, nrhs = 1024, 300, 2
    A, _ = factored_c64(D, h, m, n)
    b = c64(m, nrhs, 5)
    return lambda: D._lib.call("dhqr_apply_qt_c64", h.raw, m, n, 0, n, p(A), m, p(b), m, nrhs, None)


def backsolve_c64(D, h):
    m, n, nrhs = 1024, 300, 2
    A, al = factored_c64(D, h, m, n)
    b = c64(m, nrhs, 5)
    return lambda: D._lib.call("dhqr_backsolve_c64", h.raw, m, n, 0, n, p(A), m, p(al), p(b), m, nrhs, None)


def qrcp(D, h):
    m, n = 1024, 300
    A = f64(D, h, m, n, 3)
    al = torch.zeros(n, dtype=torch.float64, device=DEV)
    jp = torch.zeros(n, dtype=torch.int64, device=DEV)
    return lambda: D._lib.call("dhqr_qrcp_f64", h.raw, m, n, p(A), m, p(al), p(jp), None)


def solve_qrcp(D, h):
    m, n, nrhs = 1024, 300, 2
    A = f64(D, h, m, n, 3)
    al = torch.zeros(n, dtype=torch.float64, device=DEV)
    jp = torch.zeros(n, dtype=torch.int64, device=DEV)
    D._lib.call("dhqr_qrcp_f64", h.raw, m, n, p(A), m, p(al), p(jp), None)
    b = f64(D, h, m, nrhs, 5)
    return lambda: D._lib.call("dhqr_solve_qrcp_f64", h.raw, m, n, n, p(A), m, p(al), p(jp), p(b), m, nrhs, None)


def partialdot(cplx):
    def make(D, h):
        a, b = (c64(4096, 1, 1)[:, 0], c64(4096, 1, 2)[:, 0]) if cplx else (f64(D, h, 4096, 1, 1)[:, 0], f64(D, h, 4096, 1, 2)[:, 0])
        out = torch.zeros(1, dtype=a.dtype, device=DEV)
        fn = "dhqr_partialdot_c64" if cplx else "dhqr_partialdot_f64"
        return lambda: D._lib.call(fn, h.raw, p(a), p(b), 10, 4000, p(out), None)
    return make


def fill_uniform(D, h):
    A = D.colmajor_empty(1000, 70, DEV)
    return lambda: D._lib.call("dhqr_fill_uniform_f64", h.raw, 7, 0, 0, 1000, 70, p(A), 1000, None)


def qr_host(D, h):
    m, n = 3072, 1536                                                  # several upload chunks at the default host_chunk
    hA = torch.empty((n, m), dtype=torch.float64).pin_memory().t()
    hA.copy_(f64(D, h, m, n, 3).cpu())
    al = torch.empty(n, dtype=torch.float64).pin_memory()
    return lambda: D._lib.call("dhqr_qr_host_f64", h.raw, m, n, C.c_void_p(hA.data_ptr()), m, C.c_void_p(al.data_ptr()), 0)


CASES = {
    "qr_nb0_wide_pairs": qr_case(1024, 512, 0),
    "qr_nb32": qr_case(1024, 300, 32),
    "qr_nb96": qr_case(1024, 300, 96),
    "qr_nb1_fused": qr_case(1024, 200, 1, fuse_house=1),
    "qr_nb1_per_column": qr_case(1024, 200, 1, fuse_house=0),
    "qr_refused_pair": refused_pair,
    "apply_qt_nrhs1": apply_case("dhqr_apply_qt_f64", 1),
    "apply_qt_nrhs3": apply_case("dhqr_apply_qt_f64", 3),
    "apply_q_nrhs1": apply_case("dhqr_apply_q_f64", 1),
    "apply_q_nrhs3": apply_case("dhqr_apply_q_f64", 3),
    "backsolve_wave": backsolve_case(1),
    "backsolve_blocks": backsolve_case(0),
    "forwardsolve_f64": adj_case("dhqr_forwardsolve_f64", False),
    "forwardsolve_c64": adj_case("dhqr_forwardsolve_c64", True),
    "solve_adj_f64": adj_case("dhqr_solve_adj_f64", False),
    "solve_adj_c64": adj_case("dhqr_solve_adj_c64", True),
    "form_q_f64": form_q_case(False),
    "form_q_c64": form_q_case(True),
    "qr_c64": qr_c64,
    "apply_qt_c64": apply_qt_c64,
    "backsolve_c64": backsolve_c64,
    "qrcp_f64": qrcp,
    "solve_qrcp_f64": solve_qrcp,
    "partialdot_f64": partialdot(False),
    "partialdot_c64": partialdot(True),
    "fill_uniform_f64": fill_uniform,
    "qr_host_f64_pinned": qr_host,
}


@pytest.mark.parametrize("case", list(CASES))
def test_profile_counts_every_launch(D, case):
    h = D.Handle(0)
    try:
        h.set_option("profile", 1)
        run = CASES[case](D, h)
        torch.cuda.synchronize()
        h.profile_reset()
        n0, redone = h.launch_count(), h.get_option("wide_redone")
        run()
        torch.cuda.synchronize()
        launched = h.launch_count() - n0
        if case == "qr_refused_pair":
            assert h.get_option("wide_redone") == redone + 1
        prof = h.profile()
        assert launched > 0
        assert all(prof), f"a profile class without a name: {sorted(prof)}"
        counts = {k: v["count"] for k, v in prof.items() if v["count"]}
        assert sum(counts.values()) == launched, f"{launched} launches, profile counts {counts}"
    finally:
        h.close()
