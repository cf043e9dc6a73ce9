"""A handle gives back all the device memory it took: create -> a fixed program over every entry point that grows workspace ->
close leaves free device memory where it was, and a dhqr_create_dist that fails leaves neither a handle nor memory behind."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
M, N = 32768, 1024          # Float64: at m = 32768 each ring of three packed-V buffers is ~107 MB
MZ, NZ = 4096, 512          # ComplexF64
HOST_CHUNK = 256            # at M x N this upload plan joins chunks after steps 2 and 4, behind catch-ups
SLACK = 16 << 20            # free memory is device-wide, so other work on the device moves it too
MiB = 1 << 20


@pytest.fixture(scope="module")
def D():
    import dhqr_b200
    assert torch.cuda.is_available()
    return dhqr_b200


def p(t):
    return C.c_void_p(t.data_ptr())


def colmajor(m, n, dtype=torch.float64, pinned=False):
    if pinned:
        return torch.empty((n, m), dtype=dtype).pin_memory().t()
    return torch.empty((n, m), dtype=dtype, device=DEV).t()


class Program:
    """Every input is allocated once and refilled in place, so the torch caching allocator holds the same memory in every cycle."""

    def __init__(self, D, h):
        self.D = D
        self.A0, self.A, self.Q = colmajor(M, N), colmajor(M, N), colmajor(M, N)
        D.fill_uniform_(self.A0, 1, handle=h)
        self.B0, self.b = colmajor(M, 3), colmajor(M, 3)
        D.fill_uniform_(self.B0, 2, handle=h)
        self.al = torch.zeros(N, dtype=torch.float64, device=DEV)
        self.jp = torch.zeros(N, dtype=torch.int64, device=DEV)
        g = torch.Generator(device=DEV).manual_seed(3)
        self.Z0 = torch.complex(torch.rand((NZ, MZ), generator=g, device=DEV, dtype=torch.float64),
                                torch.rand((NZ, MZ), generator=g, device=DEV, dtype=torch.float64)).t()
        self.Z, self.QZ = colmajor(MZ, NZ, torch.complex128), colmajor(MZ, NZ, torch.complex128)
        self.zal = torch.zeros(NZ, dtype=torch.complex128, device=DEV)
        self.hA = colmajor(M, N, pinned=True)
        self.hal = torch.empty(N, dtype=torch.float64).pin_memory()
        bounds, join = D.plan_host_upload(M, N, 128, chunk=HOST_CHUNK)
        assert len(bounds) > 2 and max(join) > 0, (bounds, join)     # the host entry runs catch-ups

    def qr(self, h, nb):
        self.A.copy_(self.A0)
        self.D._lib.call("dhqr_qr_f64", h.raw, M, N, 0, N, p(self.A), M, p(self.al), nb, None)

    def run(self, h):
        call = self.D._lib.call
        self.qr(h, 0)                                                  # look-ahead with panel pairs
        self.qr(h, 64)
        for nrhs in (1, 3):                                            # ldiv
            self.b.copy_(self.B0)
            call("dhqr_solve_f64", h.raw, M, N, 0, N, p(self.A), M, p(self.al), p(self.b), M, nrhs, None)
        call("dhqr_form_q_f64", h.raw, M, N, p(self.A), M, p(self.Q), M, None)
        self.b.copy_(self.B0)
        call("dhqr_solve_adj_f64", h.raw, M, N, p(self.A), M, p(self.al), p(self.b), M, 3, None)
        self.Z.copy_(self.Z0)
        call("dhqr_qr_c64", h.raw, MZ, NZ, 0, NZ, p(self.Z), MZ, p(self.zal), None)
        call("dhqr_form_q_c64", h.raw, MZ, NZ, p(self.Z), MZ, p(self.QZ), MZ, None)
        self.A.copy_(self.A0)
        call("dhqr_qrcp_f64", h.raw, M, N, p(self.A), M, p(self.al), p(self.jp), None)
        self.hA.copy_(self.A0)
        h.set_option("host_chunk", HOST_CHUNK)
        call("dhqr_qr_host_f64", h.raw, M, N, p(self.hA), M, p(self.hal), 0)
        # the traces keep events and buffers in the handle until the next traced call or the handle's end
        h.set_option("profile", 1)
        self.qr(h, 0)
        h.set_option("profile", 0)                                     # the look-ahead schedule runs only without it
        h.set_option("chain_wait_trace", 1)
        self.qr(h, 0)
        h.set_option("panel_trace", 1)
        self.qr(h, 64)
        torch.cuda.synchronize()


def free_bytes():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_handle_returns_its_device_memory(D):
    h = D.Handle(0)
    try:
        prog = Program(D, h)
        prog.run(h)                                                    # warm-up: modules loaded, torch cache filled
    finally:
        h.close()
    base = free_bytes()
    drift = []
    for _ in range(3):
        h = D.Handle(0)
        try:
            prog.run(h)
        finally:
            h.close()
        drift.append(base - free_bytes())
    assert all(d <= SLACK for d in drift), "free memory below its baseline after each cycle: " + \
        ", ".join(f"{d / MiB:.1f} MiB" for d in drift)


def test_failed_dist_create_leaves_nothing(tmp_path):
    # In a process of its own: a process that already loaded NCCL (e.g. torch.distributed) would go on to ncclCommInitRank.
    code = textwrap.dedent(f"""
        import ctypes as C, sys
        sys.path.insert(0, {ROOT!r})
        import torch
        import dhqr_b200 as D
        lib = D._lib.load()
        h = C.c_void_p()
        assert lib.dhqr_create(C.byref(h), 0) == 0
        lib.dhqr_destroy(h)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        h = C.c_void_p()
        uid = C.create_string_buffer(128)
        rc = lib.dhqr_create_dist(C.byref(h), 0, C.cast(uid, C.c_void_p), 0, 2)
        torch.cuda.synchronize()
        print(rc, h.value, free0 - torch.cuda.mem_get_info()[0])
    """)
    env = dict(os.environ, DHQR_NCCL_LIBRARY=str(tmp_path / "missing" / "libnccl.so.2"))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    rc, h, drift = out.stdout.split()[-3:]
    assert int(rc) == 2001
    assert h == "None"                                                 # *h untouched (ctypes shows NULL as None)
    assert abs(int(drift)) < 2 * MiB, f"free memory moved by {int(drift)} B"
