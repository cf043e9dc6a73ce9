"""Host-side mirror of DistributedHouseholderQR.jl's interface over the libdhqr.so C-ABI.

Julia is not available in this image, so the host side is Python; names, argument meaning and
mutation/aliasing behaviour follow the reference (S:n = src/DistributedHouseholderQR.jl:n):

    qr_(A)                        qr!(A)                                  S:311-315
    H.ldiv(b) / ldiv(H, b)        H \\ b                                   S:317-321
    householder_(A, alpha)        householder!(A, alpha)                  S:113-120
    solve_householder_(b, A, α)   solve_householder!(b, H, alpha)         S:284-294
    partialdot(a, b, rng)         partialdot(a, b, is, ::Type{<:Real})    S:42-49
    alphafactor(x)                alphafactor(x::Real)                    S:8
    ColumnBlockMatrix             DArray with a (1,P) process grid        T:71 (test/runtests.jl)
    LocalColumnBlock              LocalColumnBlock{Al, dj, colrange}      S:26-40

Matrices are column-major float64, like a Julia Matrix: CUDA tensors of shape (m, n) with strides
(1, lda) (use ``colmajor_empty`` / ``to_colmajor``), or Fortran-ordered numpy arrays for the host path.
PyTorch supplies device memory, streams and torch.distributed; all arithmetic happens in libdhqr.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _lib


# --------------------------------------------------------------------------------------------
# handles
# --------------------------------------------------------------------------------------------
class Handle:
    """Owns a dhqr_handle (workspace, grid-barrier words, NCCL communicator)."""

    def __init__(self, device: int = 0, *, unique_id: Optional[bytes] = None, rank: int = 0, nranks: int = 1):
        self._h = C.c_void_p()
        self.device, self.rank, self.nranks = int(device), int(rank), int(nranks)
        if nranks > 1:
            buf = C.create_string_buffer(unique_id, 128)
            _lib.call("dhqr_create_dist", C.byref(self._h), self.device, C.cast(buf, C.c_void_p), rank, nranks)
        else:
            _lib.call("dhqr_create", C.byref(self._h), self.device)

    @property
    def raw(self) -> C.c_void_p:
        if not self._h:
            raise RuntimeError("handle destroyed")
        return self._h

    def set_option(self, key: str, value: int) -> None:
        _lib.call("dhqr_set_option", self.raw, key.encode(), int(value))

    def get_option(self, key: str) -> int:
        v = C.c_int64()
        _lib.call("dhqr_get_option", self.raw, key.encode(), C.byref(v))
        return int(v.value)

    def launch_count(self) -> int:
        v = C.c_int64()
        _lib.call("dhqr_launch_count", self.raw, C.byref(v))
        return int(v.value)

    def profile_reset(self) -> None:
        _lib.call("dhqr_profile_reset", self.raw)

    def profile(self) -> dict:
        """{kernel class: {"ms", "count", "work"}} accumulated since profile_reset() (option "profile" = 1)."""
        out, i = {}, 0
        lib = _lib.load()
        while True:
            name = C.create_string_buffer(64)
            ms, cnt, work = C.c_double(), C.c_int64(), C.c_double()
            rc = lib.dhqr_profile_get(self.raw, i, name, 64, C.byref(ms), C.byref(cnt), C.byref(work))
            if rc == -2:
                break
            if rc != 0:
                raise _lib.DhqrError("dhqr_profile_get", rc, lib.dhqr_last_error().decode())
            out[name.value.decode()] = {"ms": ms.value, "count": cnt.value, "work": work.value}
            i += 1
        return out

    def close(self) -> None:
        if self._h:
            _lib.load().dhqr_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_handles: dict = {}
_dist_handle: Optional[Handle] = None


def default_handle(device: Optional[int] = None) -> Handle:
    if _dist_handle is not None and (device is None or device == _dist_handle.device):
        return _dist_handle
    if device is None:
        device = torch.cuda.current_device()
    if device not in _default_handles:
        _default_handles[device] = Handle(device)
    return _default_handles[device]


def init_distributed(device: Optional[int] = None, group=None) -> Handle:
    """One process per GPU: build the library's NCCL communicator over the ranks of ``group``.

    torch.distributed is only the plumbing here (ships the NCCL unique id); the factorisation's own
    exchange steps are issued inside libdhqr.so."""
    global _dist_handle
    import torch.distributed as dist
    rank, nranks = dist.get_rank(group), dist.get_world_size(group)
    if device is None:
        device = torch.cuda.current_device()
    uid = bytearray(128)
    if rank == 0:
        buf = C.create_string_buffer(128)
        _lib.call("dhqr_nccl_unique_id", C.cast(buf, C.c_void_p))
        uid = bytearray(buf.raw)
    obj = [bytes(uid)]
    dist.broadcast_object_list(obj, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    _dist_handle = Handle(device, unique_id=obj[0], rank=rank, nranks=nranks)
    return _dist_handle


def shutdown_distributed() -> None:
    global _dist_handle
    if _dist_handle is not None:
        _dist_handle.close()
        _dist_handle = None


# --------------------------------------------------------------------------------------------
# layout helpers
# --------------------------------------------------------------------------------------------
def colmajor_empty(m: int, n: int, device="cuda", lda: Optional[int] = None, dtype=torch.float64) -> torch.Tensor:
    """(m, n) float64 (or complex128) tensor stored column-major with leading dimension lda (default m)."""
    lda = max(int(lda or m), 1)
    base = torch.empty((max(n, 0), lda), dtype=dtype, device=device)
    return base.t()[:m, :]


def to_colmajor(x, device="cuda") -> torch.Tensor:
    t = torch.as_tensor(x)
    t = t.to(torch.complex128 if t.is_complex() else torch.float64)
    out = colmajor_empty(t.shape[0], t.shape[1], device, dtype=t.dtype)
    out.copy_(t)
    return out


def _sfx(t: torch.Tensor) -> str:
    """C-ABI suffix for the element type: Float64 -> f64, ComplexF64 -> c64 (the reference's two element types, T:43)."""
    if t.dtype == torch.float64:
        return "f64"
    if t.dtype == torch.complex128:
        return "c64"
    raise TypeError("Float64 or ComplexF64 only (float64 / complex128), like the reference's tests (T:43)")


def _lda(A: torch.Tensor) -> int:
    m, n = A.shape
    _sfx(A)
    if m > 1 and A.stride(0) != 1:
        raise ValueError("matrix must be column-major: stride(0) == 1 (see colmajor_empty/to_colmajor)")
    lda = A.stride(1) if n > 1 else max(m, 1)
    if lda < max(m, 1):
        raise ValueError("leading dimension smaller than the row count")
    return int(lda)


def _stream_ptr(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def alphafactor(x):
    """alphafactor(x::Real) = -sign(x) (S:8);  alphafactor(x::Complex) = -exp(im * angle(x)) (S:9)."""
    if isinstance(x, complex) or np.iscomplexobj(x):
        return complex(-np.exp(1j * np.angle(x)))
    return -float(np.sign(x))


def splits(nranks: int, n: int):
    """Default DArray column distribution (DistributedArrays 0.6.7 defaultdist): even chunks, the
    remainder spread over the first blocks.  Returns the P+1 boundaries."""
    base, rem = divmod(n, nranks)
    b = [0]
    for p in range(nranks):
        b.append(b[-1] + base + (1 if p < rem else 0))
    return b


def balanced_splits(nranks: int, n: int, rule: str = "trailing"):
    """Load-balanced contiguous column splits; the reference carries two of them next to its DArray test (unused there:
    the code that would consume them, T:67-68, is commented out).

    rule="trailing": splits(np, N, p) = round((N / sqrt(np)) * sqrt(p))  (T:35) — column c is updated by the c reflectors
                     to its left, so equal work means equal areas under that ramp: early ranks get MORE columns.  This is
                     the split that evens out the trailing-update flops of the right-looking factorisation.
    rule="upstream": splits(np, N, p) = round(N * (1 - sqrt((np - p) / np)))  (T:36, the definition left active upstream) —
                     the mirror image (early ranks get fewer columns).

    Any contiguous, ascending partition is accepted by the C-ABI; pass the result as ``boundaries`` to
    ColumnBlockMatrix.from_function."""
    if rule == "trailing":
        b = [int(round(n * (p / nranks) ** 0.5)) for p in range(nranks + 1)]
    elif rule == "upstream":
        b = [int(round(n * (1.0 - ((nranks - p) / nranks) ** 0.5))) for p in range(nranks + 1)]
    else:
        raise ValueError("rule must be 'trailing' or 'upstream'")
    b[0], b[-1] = 0, n
    for p in range(1, nranks + 1):          # monotone even for tiny n
        b[p] = max(b[p], b[p - 1])
    return b


@dataclass
class LocalColumnBlock:
    """LocalColumnBlock{Al, dj, colrange} (S:26-40): local storage + global column offset."""
    Al: torch.Tensor
    dj: int            # Δj: global index of the first local column (0-based)
    colrange: range

    def global_col(self, j: int) -> torch.Tensor:
        return self.Al[:, j - self.dj]


class ColumnBlockMatrix:
    """The (1, P) DArray of the reference (T:71): every rank holds all m rows of a contiguous block
    of columns (asserted at S:33).  ``local`` is this rank's block, column-major on its GPU."""

    def __init__(self, local: torch.Tensor, n_global: int, col0: int, handle: Optional[Handle] = None):
        self.local, self.n_global, self.col0 = local, int(n_global), int(col0)
        self.handle = handle or default_handle(local.device.index)
        _lda(local)

    @property
    def shape(self):
        return (self.local.shape[0], self.n_global)

    def localblock(self) -> LocalColumnBlock:
        return LocalColumnBlock(self.local, self.col0, range(self.col0, self.col0 + self.local.shape[1]))

    @classmethod
    def from_function(cls, fill, m: int, n: int, handle: Handle, boundaries=None):
        """DArray(ij -> A[ij...], (m,n), workers(), (1, nworkers())) (T:71): ``fill(col0, ncols)``
        returns the (m, ncols) block for this rank.  ``boundaries`` (P+1 ascending column boundaries, same on every rank)
        overrides the default distribution, e.g. ``balanced_splits(P, n)`` (T:35-36)."""
        b = list(boundaries) if boundaries is not None else splits(handle.nranks, n)
        if len(b) != handle.nranks + 1 or b[0] != 0 or b[-1] != n or any(b[i] > b[i + 1] for i in range(handle.nranks)):
            raise ValueError(f"boundaries must be {handle.nranks + 1} ascending values from 0 to n={n}, got {b}")
        c0, c1 = b[handle.rank], b[handle.rank + 1]
        return cls(to_colmajor(fill(c0, c1 - c0), device=f"cuda:{handle.device}"), n, c0, handle)


# --------------------------------------------------------------------------------------------
# qr! and \
# --------------------------------------------------------------------------------------------
class DistributedHouseholderQRStruct:
    """DistributedHouseholderQRStruct{A, α} (S:296-309).  ``.A`` aliases the caller's storage
    (qr! works in place); ``.α`` (also ``.alpha``) is freshly allocated, length size(A, 2)."""

    def __init__(self, A, alpha, handle: Optional[Handle] = None):
        self.A = A
        self.α = alpha
        self.handle = handle

    @property
    def alpha(self):
        return self.α

    def ldiv(self, b):
        return ldiv(self, b)

    solve = ldiv

    def ldiv_adjoint(self, c):
        return ldiv_adjoint(self, c)


def _dev_args(A):
    if isinstance(A, ColumnBlockMatrix):
        return A.local, A.n_global, A.col0, A.handle
    return A, A.shape[1], 0, default_handle(A.device.index)


def plan_host_upload(m: int, n: int, nb: int = 128, chunk: int = 512, first: int = 0, h2d_gbs: int = 50, tflops: int = 27,
                     chain_us: int = 300):
    """The upload plan of the pipelined host entry (dhqr_plan_host_upload; pure host logic, needs no GPU): (bounds, join) with
    chunk j = columns [bounds[j], bounds[j+1]) joining the trailing matrix at step join[j] of the look-ahead schedule."""
    cap = max(2, n // max(nb, 1) + 3)
    bounds = (C.c_int64 * cap)()
    join = (C.c_int * cap)()
    nch = C.c_int()
    _lib.call("dhqr_plan_host_upload", int(m), int(n), int(nb), int(chunk), int(first), int(h2d_gbs), int(tflops), int(chain_us), cap,
              bounds, join, C.byref(nch))
    k = nch.value
    return [int(bounds[j]) for j in range(k + 1)], [int(join[j]) for j in range(k)]


def householder_(A, alpha, nb: int = 0, handle: Optional[Handle] = None):
    """householder!(A, α) (S:113-120): factor in place, α <- diag(R).  Returns (A, α)."""
    loc, n, col0, h = _dev_args(A)
    h = handle or h
    m = loc.shape[0]
    if alpha.dtype != loc.dtype:
        raise TypeError("alpha must have the element type of A")
    with torch.cuda.device(loc.device):
        if _sfx(loc) == "c64":
            _lib.call("dhqr_qr_c64", h.raw, m, n, col0, loc.shape[1], C.c_void_p(loc.data_ptr()), _lda(loc),
                      C.c_void_p(alpha.data_ptr()), _stream_ptr(loc.device))
        else:
            _lib.call("dhqr_qr_f64", h.raw, m, n, col0, loc.shape[1], C.c_void_p(loc.data_ptr()), _lda(loc),
                      C.c_void_p(alpha.data_ptr()), int(nb), _stream_ptr(loc.device))
    return A, alpha


def qr_(A, nb: int = 0, handle: Optional[Handle] = None) -> DistributedHouseholderQRStruct:
    """qr!(A) (S:311-315).  ``A``: column-major CUDA tensor, ColumnBlockMatrix, or a Fortran-ordered
    numpy array (host path: H2D, factor, D2H inside the call).  nb: 0 = default blocked (128),
    1 = unblocked reference-style column loop, else panel width (multiple of 32)."""
    if isinstance(A, np.ndarray):
        if not (A.dtype == np.float64 and A.ndim == 2 and A.flags.f_contiguous):
            raise ValueError("host matrix must be a Fortran-ordered float64 array")
        h = handle or default_handle()
        m, n = A.shape
        alpha = np.zeros(n)
        _lib.call("dhqr_qr_host_f64", h.raw, m, n, C.c_void_p(A.ctypes.data), max(A.strides[1] // 8, 1) if n > 0 else max(m, 1),
                  C.c_void_p(alpha.ctypes.data), int(nb))
        return DistributedHouseholderQRStruct(A, alpha, h)
    loc, n, _, h = _dev_args(A)
    h = handle or h
    alpha = torch.zeros(n, dtype=loc.dtype, device=loc.device)                # S:302 / S:307
    householder_(A, alpha, nb, h)                                             # S:313
    return DistributedHouseholderQRStruct(A, alpha, h)


qr_bang = qr_


def solve_householder_(b: torch.Tensor, A, alpha: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """solve_householder!(b, H, α) (S:284-294): b <- Q'b, back-substitute, return b[1:n] (a view, S:293).
    ``b``: length-m vector or (m, k) column-major block of right-hand sides; overwritten."""
    loc, n, col0, h = _dev_args(A)
    h = handle or h
    m = loc.shape[0]
    ldb, nrhs = _rhs_args(b, m, loc.dtype)
    with torch.cuda.device(loc.device):
        _lib.call("dhqr_solve_" + _sfx(loc), h.raw, m, n, col0, loc.shape[1], C.c_void_p(loc.data_ptr()), _lda(loc),
                  C.c_void_p(alpha.data_ptr()), C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(loc.device))
    return b[:n]


def _rhs_args(b: torch.Tensor, m: int, dtype=torch.float64):
    if b.dtype != dtype:
        raise TypeError(f"b must have the element type of A ({dtype})")
    if b.dim() not in (1, 2) or b.shape[0] != m:
        raise ValueError(f"b must have {m} rows (a length-m vector or an (m, k) column-major block)")
    if b.dim() == 1:
        if not b.is_contiguous():
            raise ValueError("b must be contiguous")
        return max(m, 1), 1
    return _lda(b), b.shape[1]


def _apply(fn: str, b: torch.Tensor, A, handle: Optional[Handle]) -> torch.Tensor:
    loc, n, col0, h = _dev_args(A)
    h = handle or h
    m = loc.shape[0]
    ldb, nrhs = _rhs_args(b, m, loc.dtype)
    with torch.cuda.device(loc.device):
        _lib.call(fn + _sfx(loc), h.raw, m, n, col0, loc.shape[1], C.c_void_p(loc.data_ptr()), _lda(loc),
                  C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(loc.device))
    return b


def apply_qt_(b: torch.Tensor, A, handle: Optional[Handle] = None) -> torch.Tensor:
    """_solve_householder1! (S:226-242): b <- H_n ... H_1 b = Q'b, in place (b: length m, or (m, k) column-major)."""
    return _apply("dhqr_apply_qt_", b, A, handle)


def apply_q_(b: torch.Tensor, A, handle: Optional[Handle] = None) -> torch.Tensor:
    """b <- H_1 ... H_n b = Q b, in place: the inverse of apply_qt_ (the reference never forms Q; this exposes the
    factorisation as an operator, SURVEY 8f-3)."""
    if (A.local if isinstance(A, ColumnBlockMatrix) else A).dtype != torch.float64:
        raise TypeError("apply_q_ is Float64 only")
    return _apply("dhqr_apply_q_", b, A, handle)


def form_q(A, out: Optional[torch.Tensor] = None, handle: Optional[Handle] = None) -> torch.Tensor:
    """The thin Q of a factorisation: the first n columns of H_1 ... H_n (numpy.linalg.qr / torch.linalg.qr mode "reduced",
    LAPACK orgqr / ungqr).  ``A`` is the factored matrix (as for apply_q_ / backsolve_), Float64 or ComplexF64.  Returns Q as an
    (m, n) column-major tensor of A's dtype: freshly allocated for ``out=None``; ``out is A`` overwrites the factorisation with Q
    (R is lost: take form_r first); any other ``out`` must be an (m, n) column-major tensor that does not overlap A.
    Single GPU: a ColumnBlockMatrix on a multi-rank handle raises the library's -1."""
    if isinstance(A, np.ndarray):
        raise TypeError("form_q works on a device-resident factorisation (a CUDA tensor), not a numpy array")
    loc, n, _, h = _dev_args(A)
    h = handle or h
    m = loc.shape[0]
    if out is A:
        out = loc
    if out is None:
        out = colmajor_empty(m, n, loc.device, dtype=loc.dtype)
    elif out is not loc:
        if out.dtype != loc.dtype or out.device != loc.device:
            raise TypeError(f"out must be a {loc.dtype} tensor on {loc.device}")
        if tuple(out.shape) != (m, n):
            raise ValueError(f"out must have shape ({m}, {n})")
    with torch.cuda.device(loc.device):
        _lib.call("dhqr_form_q_" + _sfx(loc), h.raw, m, n, C.c_void_p(loc.data_ptr()), _lda(loc), C.c_void_p(out.data_ptr()),
                  _lda(out), _stream_ptr(loc.device))
    return out


def form_r(A, alpha: torch.Tensor) -> torch.Tensor:
    """R = triu(A[:n], 1) + diag(alpha) as an (n, n) tensor, from the factored matrix and alpha (torch, no kernel of its own).
    Take it before an in-place form_q, which overwrites R's rows."""
    loc = A.local if isinstance(A, ColumnBlockMatrix) else A
    n = loc.shape[1]
    return torch.triu(loc[:n], 1) + torch.diag(alpha.to(loc.dtype))


def backsolve_(b: torch.Tensor, A, alpha: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """_solve_householder2! (S:256-282): b[0:n] <- R^{-1} b[0:n] with R = triu(A,1) + diag(alpha); returns b[0:n]."""
    loc, n, col0, h = _dev_args(A)
    h = handle or h
    m = loc.shape[0]
    ldb, nrhs = _rhs_args(b, m, loc.dtype)
    with torch.cuda.device(loc.device):
        _lib.call("dhqr_backsolve_" + _sfx(loc), h.raw, m, n, col0, loc.shape[1], C.c_void_p(loc.data_ptr()), _lda(loc),
                  C.c_void_p(alpha.data_ptr()), C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(loc.device))
    return b[:n]


def _adj(fn: str, b: torch.Tensor, A, alpha: torch.Tensor, handle: Optional[Handle]) -> int:
    if isinstance(A, np.ndarray):
        raise TypeError("the adjoint solves work on a device-resident factorisation (a CUDA tensor), not a numpy array")
    loc, n, _, h = _dev_args(A)
    h = handle or h
    m = loc.shape[0]
    if alpha.dtype != loc.dtype:
        raise TypeError("alpha must have the element type of A")
    ldb, nrhs = _rhs_args(b, m, loc.dtype)
    with torch.cuda.device(loc.device):
        _lib.call(fn + _sfx(loc), h.raw, m, n, C.c_void_p(loc.data_ptr()), _lda(loc), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(loc.device))
    return n


def forwardsolve_(b: torch.Tensor, A, alpha: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """b[0:n] <- R^{-H} b[0:n] (R^{-T} for Float64) with R = triu(A,1) + diag(alpha): forward substitution with the lower-triangular
    R^H, the adjoint of backsolve_.  ``b``: length-m vector or (m, k) column-major block; rows n..m-1 are left as they are.
    Returns b[0:n].  Single GPU."""
    return b[:_adj("dhqr_forwardsolve_", b, A, alpha, handle)]


def solve_adjoint_(b: torch.Tensor, A, alpha: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """The minimum-norm solution of A^H y = c (LAPACK ?gels, TRANS = 'C'): rows [0, n) of ``b`` hold c on entry, all m rows hold
    y = Q [R^{-H} c; 0] on return.  ``b``: length-m vector or (m, k) column-major block.  Returns b.  Single GPU."""
    _adj("dhqr_solve_adj_", b, A, alpha, handle)
    return b


def ldiv_adjoint(H: DistributedHouseholderQRStruct, c):
    """H^H \\ c: the minimum-norm solution y of A^H y = c for the factored A (length n, or (n, k)).  Neither H nor c is modified;
    returns a new length-m vector or (m, k) tensor."""
    if isinstance(H.A, np.ndarray):
        raise TypeError("ldiv_adjoint works on a device-resident factorisation (a CUDA tensor), not a numpy array")
    loc = H.A.local if isinstance(H.A, ColumnBlockMatrix) else H.A
    m, n = loc.shape[0], H.α.shape[0]
    c = torch.as_tensor(c)
    if c.is_complex() != loc.is_complex():
        raise TypeError(f"c must have the element type of A ({loc.dtype})")
    if c.dim() not in (1, 2) or c.shape[0] != n:
        raise ValueError(f"c must have {n} rows (a length-n vector or an (n, k) block)")
    if c.dim() == 1:
        y = torch.empty(m, dtype=loc.dtype, device=loc.device)
        y[:n] = c.to(device=loc.device, dtype=loc.dtype)
    else:
        y = colmajor_empty(m, c.shape[1], loc.device, dtype=loc.dtype)
        y[:n] = c.to(device=loc.device, dtype=loc.dtype)
    return solve_adjoint_(y, H.A, H.α, H.handle)


def ldiv(H: DistributedHouseholderQRStruct, b):
    """H \\ b (S:317-321): neither H nor b is modified; returns a new length-n vector."""
    if isinstance(H.A, np.ndarray):
        m, n = H.A.shape
        bb = np.ascontiguousarray(b, dtype=np.float64)
        if bb.ndim != 1 or bb.shape[0] != m:
            raise ValueError(f"b must be a length-{m} vector")
        x = np.zeros(n)
        _lib.call("dhqr_ldiv_host_f64", H.handle.raw, m, n, C.c_void_p(H.A.ctypes.data), max(H.A.strides[1] // 8, 1),
                  C.c_void_p(H.α.ctypes.data), C.c_void_p(bb.ctypes.data), C.c_void_p(x.ctypes.data))
        return x
    loc = H.A.local if isinstance(H.A, ColumnBlockMatrix) else H.A
    if b.dim() == 1:
        s = b.to(device=loc.device, dtype=loc.dtype).clone()                      # S:318
    else:
        s = to_colmajor(b, device=loc.device)
    x = solve_householder_(s, H.A, H.α, H.handle)                                # S:319
    return x.clone()                                                              # S:320


# --------------------------------------------------------------------------------------------
# QR with column pivoting (LAPACK dgeqp3) and the basic least-squares solution (dgelsy without the complete orthogonal
# decomposition); scipy.linalg.qr(pivoting=True) / Julia's qr(A, ColumnNorm())
# --------------------------------------------------------------------------------------------
def _rhs_copy(b, A: torch.Tensor) -> torch.Tensor:
    """A fresh copy of ``b`` (length m, or (m, k)) on A's device for the pivoted solves: a vector takes A's dtype, a block is made
    column-major, and a real block is promoted to complex128 for a ComplexF64 factorisation."""
    if b.dim() == 1:
        return b.to(device=A.device, dtype=A.dtype).clone()
    if A.is_complex():
        out = colmajor_empty(b.shape[0], b.shape[1], A.device, dtype=A.dtype)
        out.copy_(torch.as_tensor(b))
        return out
    return to_colmajor(b, device=A.device)


class PivotedHouseholderQRStruct:
    """A P = Q R from ``qrcp_``: ``.A`` (the caller's storage, factored in place) and ``.α`` (``.alpha``) are the factorisation of
    ``A[:, p]`` in the library's storage format, so every other entry point (apply_qt_, apply_q_, backsolve_, form_q,
    forwardsolve_) takes them as that; ``.p`` is an int64 device tensor, ``p[k]`` = original index of the k-th column."""

    def __init__(self, A, alpha, p, handle: Optional[Handle] = None):
        self.A = A
        self.α = alpha
        self.p = p
        self.handle = handle

    @property
    def alpha(self):
        return self.α

    def rank(self, rcond: Optional[float] = None) -> int:
        """Numerical rank: the first k with |α_k| <= rcond |α_0| (n if there is none).  Default rcond = max(m, n) eps.  Reads α,
        so it synchronises with the stream the factorisation ran on."""
        m, n = self.A.shape[0], self.α.shape[0]
        if n == 0:
            return 0
        if rcond is None:
            rcond = max(m, n) * float(np.finfo(np.float64).eps)
        a = self.α.abs().cpu().numpy()
        small = np.nonzero(~(a > rcond * a[0]))[0]
        return int(small[0]) if small.size else n

    def ldiv(self, b, rcond: Optional[float] = None):
        """The basic solution x of min ||A x - b|| at rank ``self.rank(rcond)``; returns (x, rank).  Neither the factorisation nor
        b is modified.  ``b``: length m, or (m, k)."""
        r = self.rank(rcond)
        loc = self.A
        s = _rhs_copy(b, loc)
        solve_qrcp_(s, self.A, self.α, self.p, r, self.handle)
        return s[:loc.shape[1]].clone(), r

    solve = ldiv

    def cod(self, rcond: Optional[float] = None) -> "CompleteOrthogonalStruct":
        """The complete orthogonal decomposition A P ~ Q1 [U' 0] Z' at rank ``self.rank(rcond)`` (DESIGN §2.8), whose ``.ldiv``
        gives the minimum-norm least-squares solution, as numpy.linalg.lstsq and LAPACK dgelsy do.  The factorisation is read,
        never modified."""
        r = self.rank(rcond)
        F, gamma = cod_(self.A, self.α, r, self.handle)
        return CompleteOrthogonalStruct(self, F, gamma, r)


class CompleteOrthogonalStruct:
    """A P ~ Q1 [U' 0] Z' from ``PivotedHouseholderQRStruct.cod``: ``.qrcp`` is the pivoted factorisation (Q1, P), ``.F`` and ``.γ``
    (``.gamma``) the factorisation R_r' = Z [U; 0] of the leading ``.rank`` rows of R, in the library's storage format (so
    form_q(F) is Z[:, :rank], and forwardsolve_ / apply_q_ take (F, γ) as any other factorisation)."""

    def __init__(self, qrcp, F, gamma, rank: int):
        self.qrcp = qrcp
        self.F = F
        self.γ = gamma
        self.rank = rank

    @property
    def gamma(self):
        return self.γ

    def ldiv(self, b):
        """The minimum-norm solution x of min ||A x - b|| at rank ``self.rank``; neither the factorisations nor b is modified.
        ``b``: length m, or (m, k).  Returns a new length-n vector or (n, k) tensor."""
        A = self.qrcp.A
        s = _rhs_copy(b, A)
        solve_cod_(s, A, self.qrcp.p, self.F, self.γ, self.rank, self.qrcp.handle)
        return s[:A.shape[1]].clone()

    solve = ldiv


def qrcp_(A: torch.Tensor, handle: Optional[Handle] = None) -> PivotedHouseholderQRStruct:
    """A P = Q R with column pivoting (LAPACK dgeqp3 / zgeqp3; scipy.linalg.qr(pivoting=True)), in place, on a column-major float64
    or complex128 CUDA tensor with n <= m (alpha has A's dtype).  Single GPU, stream-ordered, no synchronisation."""
    if not isinstance(A, torch.Tensor) or not A.is_cuda:
        raise TypeError("qrcp_ works on a column-major float64 or complex128 CUDA tensor")
    if A.dtype not in (torch.float64, torch.complex128):
        raise TypeError("qrcp_ takes Float64 or ComplexF64 (float64 / complex128) only")
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    alpha = torch.zeros(n, dtype=A.dtype, device=A.device)
    p = torch.zeros(n, dtype=torch.int64, device=A.device)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_qrcp_" + _sfx(A), h.raw, m, n, C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(p.data_ptr()), _stream_ptr(A.device))
    return PivotedHouseholderQRStruct(A, alpha, p, h)


def solve_qrcp_(b: torch.Tensor, A: torch.Tensor, alpha: torch.Tensor, p: torch.Tensor, rank: int,
                handle: Optional[Handle] = None) -> torch.Tensor:
    """x = P [R11^{-1} (Q^H b)[0:rank]; 0], the basic solution at the given rank, from a factorisation made by ``qrcp_`` (Float64
    or ComplexF64).  ``b``:
    length m, or (m, k) column-major; on return b[0:n] = x (returned as a view) and rows n..m-1 hold rows n..m-1 of
    H_rank ... H_1 b."""
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    sfx = _sfx(A)
    if alpha.dtype != A.dtype or p.dtype != torch.int64:
        raise TypeError("alpha must have the element type of A and p must be int64")
    ldb, nrhs = _rhs_args(b, m, A.dtype)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_solve_qrcp_" + sfx, h.raw, m, n, int(rank), C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(p.data_ptr()), C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(A.device))
    return b[:n]


def cod_(A: torch.Tensor, alpha: torch.Tensor, rank: int, handle: Optional[Handle] = None):
    """The second factorisation of the complete orthogonal decomposition at the given rank, from a factorisation made by
    ``qrcp_``: R_r^H = Z [U; 0] with R_r = rows [0, rank) of R = triu(A, 1) + diag(alpha).  Returns (F, γ): F a fresh (n, rank)
    column-major tensor of A's dtype in the library's storage format, γ = diag(U).  A and alpha are read, never written.  Float64:
    synchronises the stream once when a 128-column panel of R_r' went through the wide chain, as qr_ does; ComplexF64 never
    synchronises."""
    if not isinstance(A, torch.Tensor) or not A.is_cuda or A.dtype not in (torch.float64, torch.complex128):
        raise TypeError("cod_ works on a column-major float64 or complex128 CUDA tensor")
    if alpha.dtype != A.dtype:
        raise TypeError("alpha must have the element type of A")
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    rank = int(rank)
    F = colmajor_empty(n, max(rank, 0), A.device, dtype=A.dtype)
    gamma = torch.zeros(max(rank, 0), dtype=A.dtype, device=A.device)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_cod_" + _sfx(A), h.raw, m, n, rank, C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(F.data_ptr() if rank > 0 else None), max(n, 1), C.c_void_p(gamma.data_ptr() if rank > 0 else None),
                  _stream_ptr(A.device))
    return F, gamma


def solve_cod_(b: torch.Tensor, A: torch.Tensor, p: torch.Tensor, F: torch.Tensor, gamma: torch.Tensor, rank: int,
               handle: Optional[Handle] = None) -> torch.Tensor:
    """x = P Z [U^{-H} (Q^H b)[0:rank]; 0], the minimum-norm solution at the given rank, from ``qrcp_``'s (A, p) and ``cod_``'s
    (F, γ) at that rank (Float64 or ComplexF64).  ``b``: length m, or (m, k) column-major; on return b[0:n] = x (returned as a view) and rows n..m-1
    hold rows n..m-1 of H_rank ... H_1 b, as in solve_qrcp_."""
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    sfx = _sfx(A)
    if p.dtype != torch.int64 or F.dtype != A.dtype or gamma.dtype != A.dtype:
        raise TypeError("p must be int64, F and gamma of the element type of A")
    rank = int(rank)
    if rank > 0 and (tuple(F.shape) != (n, rank) or tuple(gamma.shape) != (rank,)):
        raise ValueError(f"F must be ({n}, {rank}) and gamma ({rank},)")
    ldb, nrhs = _rhs_args(b, m, A.dtype)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_solve_cod_" + sfx, h.raw, m, n, rank, C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(p.data_ptr()),
                  C.c_void_p(F.data_ptr() if rank > 0 else None), _lda(F) if rank > 0 else max(n, 1),
                  C.c_void_p(gamma.data_ptr() if rank > 0 else None), C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(A.device))
    return b[:n]


def partialdot(a: torch.Tensor, b: torch.Tensor, rng, handle: Optional[Handle] = None):
    """partialdot(a, b, is, ::Type{<:Real}) (S:42-49) / ::Type{<:Complex} (S:51-59: sum conj(a[i]) b[i]); ``rng`` is a
    0-based Python range."""
    h = handle or default_handle(a.device.index)
    if a.dtype != b.dtype:
        raise TypeError("a and b must have the same element type")
    i0, i1 = (rng.start, rng.stop) if len(rng) else (0, 0)
    out = torch.zeros(1, dtype=a.dtype, device=a.device)
    with torch.cuda.device(a.device):
        _lib.call("dhqr_partialdot_" + _sfx(a), h.raw, C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), i0, i1,
                  C.c_void_p(out.data_ptr()), _stream_ptr(a.device))
    v = out.item()
    return complex(v) if a.is_complex() else float(v)


def fill_uniform_(A: torch.Tensor, seed: int, i0: int = 0, j0: int = 0, handle: Optional[Handle] = None) -> torch.Tensor:
    """A[i,j] = U[0,1) keyed on (seed, i0+i, j0+j): the synthetic rand(m,n) of T:45-46, bit-identical
    on every rank and in the CPU oracle."""
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    with torch.cuda.device(A.device):
        _lib.call("dhqr_fill_uniform_f64", h.raw, seed, i0, j0, m, n, C.c_void_p(A.data_ptr()), _lda(A),
                  _stream_ptr(A.device))
    return A


# --------------------------------------------------------------------------------------------
# new rows into an existing factorisation (LAPACK dtpqrt / dtpmqrt), DESIGN §2.10, and rows out of it again (§2.11)
# --------------------------------------------------------------------------------------------
class _RowReflectors:
    """The reflectors of an append or a downdate: ``.B`` holds their tails V2 (k x n, the caller's block, overwritten) and
    ``.vtop`` their tops."""

    def __init__(self, B, vtop, handle: Handle):
        self.B = B
        self.vtop = vtop
        self.handle = handle

    def _apply(self, fn: str, c: torch.Tensor, e: torch.Tensor):
        k, n = self.B.shape
        ldc, nrhs = _rhs_args(c, n)
        lde, nrhs_e = _rhs_args(e, k)
        if nrhs != nrhs_e:
            raise ValueError("c and e must have the same number of right-hand sides")
        with torch.cuda.device(self.B.device):
            _lib.call(fn, self.handle.raw, n, k, C.c_void_p(self.B.data_ptr()), _lda(self.B), C.c_void_p(self.vtop.data_ptr()),
                      C.c_void_p(c.data_ptr()), ldc, C.c_void_p(e.data_ptr()), lde, nrhs, _stream_ptr(self.B.device))
        return c, e


class AppendedRows(_RowReflectors):
    """[R; B] = Q~ [R'; 0] from ``append_rows_``: ``.B`` holds the reflector tails V2 (k x n, the caller's block, overwritten) and
    ``.vtop`` their tops, so H~_j = I - v~_j v~_j' with v~_j = vtop[j] on row j of R and B[:, j] on the new rows."""

    def apply_qt_(self, c: torch.Tensor, e: torch.Tensor):
        """[c; e] <- Q~' [c; e] in place: c has n rows, e has k rows (vectors, or column-major blocks of equal width)."""
        return self._apply("dhqr_apply_qt_append_f64", c, e)

    def apply_q_(self, c: torch.Tensor, e: torch.Tensor):
        """[c; e] <- Q~ [c; e] in place, the inverse of apply_qt_."""
        return self._apply("dhqr_apply_q_append_f64", c, e)


class DowndatedRows(_RowReflectors):
    """Theta [R; Z] = [R'; 0] from ``downdate_rows_``: ``.B`` holds the hyperbolic reflector tails V2 (k x n, the caller's block,
    overwritten), ``.vtop`` their tops, so Theta_j = I - v~_j v~_j' J with J = diag(I_n, -I_k).  ``.info`` is a one-element int64
    CUDA tensor: 0, or the 1-based column at which the removal proved impossible (R'R - Z'Z not positive definite); reading it
    synchronises with the device."""

    def __init__(self, B, vtop, info, handle: Handle):
        super().__init__(B, vtop, handle)
        self.info = info

    def apply_(self, c: torch.Tensor, e: torch.Tensor):
        """[c; e] <- Theta [c; e] in place: c = (Q'b)[0:n] (n rows) and e the removed rows' right-hand sides (k rows) become c' and
        e'; x' = R'^{-1} c', and the residual sum of squares drops by ||e'||^2."""
        return self._apply("dhqr_apply_downdate_f64", c, e)


def _row_block_args(H, B: torch.Tensor, handle: Optional[Handle], what: str):
    A, alpha = (H.A, H.α) if isinstance(H, DistributedHouseholderQRStruct) else H
    if isinstance(A, ColumnBlockMatrix) or not isinstance(A, torch.Tensor) or not A.is_cuda:
        raise TypeError(f"{what} works on a single-GPU factorisation held in a CUDA tensor")
    if A.dtype != torch.float64 or alpha.dtype != torch.float64 or B.dtype != torch.float64:
        raise TypeError(f"{what} is Float64 only")
    n = alpha.shape[0]
    if A.shape[1] != n or A.shape[0] < n:
        raise ValueError("A must have len(alpha) columns and at least as many rows")
    if B.dim() != 2 or B.shape[1] != n:
        raise ValueError(f"B must be a (k, {n}) column-major block")
    h = handle or getattr(H, "handle", None) or default_handle(A.device.index)
    return A, alpha, n, B.shape[0], h


def append_rows_(H, B: torch.Tensor, handle: Optional[Handle] = None) -> AppendedRows:
    """Fold the k new rows ``B`` (a column-major float64 CUDA tensor, k x n) into the factorisation ``H`` (a single-GPU
    DistributedHouseholderQRStruct, or a pair (A, α)): afterwards (H.A, H.α) hold R' of [R; B] = Q~ [R'; 0] in A's strict upper
    triangle and α, while A's diagonal and lower trapezoid (the original reflectors) are left as they are.  ``B`` is overwritten
    with the reflector tails.  k may not exceed the handle's option "append_max_rows" (StreamingLeastSquares splits larger
    blocks).  Stream-ordered, no synchronisation."""
    A, alpha, n, k, h = _row_block_args(H, B, handle, "append_rows_")
    vtop = torch.zeros(n, dtype=torch.float64, device=A.device)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_qr_append_f64", h.raw, n, k, C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(B.data_ptr()), _lda(B), C.c_void_p(vtop.data_ptr()), _stream_ptr(A.device))
    return AppendedRows(B, vtop, h)


def downdate_rows_(H, Z: torch.Tensor, handle: Optional[Handle] = None) -> DowndatedRows:
    """Remove the k rows ``Z`` (a column-major float64 CUDA tensor, k x n) from the factorisation ``H`` (as for append_rows_):
    afterwards (H.A, H.α) hold R' with R''R' = R'R - Z'Z in A's strict upper triangle and α; A's diagonal and lower trapezoid are
    left as they are.  ``Z`` is overwritten with the reflector tails.  Only rows that were folded into R may be removed: when the
    removal is impossible, ``.info`` names the first column that showed it, and from that column on α is NaN.  k is capped by
    "append_max_rows" as for the append.  Stream-ordered, no synchronisation."""
    A, alpha, n, k, h = _row_block_args(H, Z, handle, "downdate_rows_")
    vtop = torch.zeros(n, dtype=torch.float64, device=A.device)
    info = torch.zeros(1, dtype=torch.int64, device=A.device)     # an n = 0 or k = 0 no-op leaves it untouched
    with torch.cuda.device(A.device):
        _lib.call("dhqr_qr_downdate_f64", h.raw, n, k, C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(Z.data_ptr()), _lda(Z), C.c_void_p(vtop.data_ptr()), C.c_void_p(info.data_ptr()), _stream_ptr(A.device))
    return DowndatedRows(Z, vtop, info, h)


class StreamingLeastSquares:
    """min ||A x - b|| for an A of any height, fed block by block: each block of rows is folded into R (starting from R = 0) and
    its right-hand sides into c = (Q'b)[0:n]; what the rotation moves out of reach adds to the residual.  Blocks above the row cap
    of one append are split.  ``add`` takes CUDA tensors or Fortran-ordered numpy arrays (uploaded); ``solve`` returns x as an
    (n, nrhs) tensor (a length-n vector for nrhs = 1).  ``remove`` takes rows out again, so ``add`` of the newest block followed
    by ``remove`` of the oldest keeps a sliding window::

        ls = StreamingLeastSquares(n)
        for A_blk, b_blk in blocks:
            ls.add(A_blk, b_blk)
            window.append((A_blk, b_blk))
            if len(window) > w:
                ls.remove(*window.pop(0))
            x = ls.solve()
    """

    def __init__(self, n: int, nrhs: int = 1, device=0, handle: Optional[Handle] = None):
        self.n, self.nrhs = int(n), int(nrhs)
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.handle = handle or default_handle(self.device.index)
        self.A = colmajor_empty(self.n, self.n, self.device)
        self.A.zero_()
        self.α = torch.zeros(self.n, dtype=torch.float64, device=self.device)
        self.c = colmajor_empty(self.n, self.nrhs, self.device)
        self.c.zero_()
        self._ss = torch.zeros(self.nrhs, dtype=torch.float64, device=self.device)
        self.rows = 0
        self._cap = self.handle.get_option("append_max_rows")

    def add(self, A_blk, b_blk) -> "StreamingLeastSquares":
        """Fold rows ``A_blk`` (k x n) with right-hand sides ``b_blk`` (length k, or k x nrhs) into the problem."""
        A_blk = torch.as_tensor(A_blk)
        b_blk = torch.as_tensor(b_blk)
        if b_blk.dim() == 1:
            b_blk = b_blk[:, None]
        k = A_blk.shape[0]
        if A_blk.dim() != 2 or A_blk.shape[1] != self.n or tuple(b_blk.shape) != (k, self.nrhs):
            raise ValueError(f"need a (k, {self.n}) block and its (k, {self.nrhs}) right-hand sides")
        for r0 in range(0, k, self._cap):
            r1 = min(k, r0 + self._cap)
            B = to_colmajor(A_blk[r0:r1], device=self.device)
            e = to_colmajor(b_blk[r0:r1], device=self.device)
            append_rows_((self.A, self.α), B, self.handle).apply_qt_(self.c, e)
            self._ss += (e * e).sum(0)
        self.rows += k
        return self

    def remove(self, A_blk, b_blk) -> "StreamingLeastSquares":
        """Take rows ``A_blk`` (k x n) with right-hand sides ``b_blk`` out of the problem again: they must be rows that were added.
        R, α and c are downdated as copies and swapped in only when every block succeeded; the call reads the downdates' status
        once (one synchronisation).  An impossible removal (the rows were never added, or the remaining rows are rank-deficient)
        raises ValueError and leaves the solver as it was."""
        A_blk = torch.as_tensor(A_blk)
        b_blk = torch.as_tensor(b_blk)
        if b_blk.dim() == 1:
            b_blk = b_blk[:, None]
        k = A_blk.shape[0]
        if A_blk.dim() != 2 or A_blk.shape[1] != self.n or tuple(b_blk.shape) != (k, self.nrhs):
            raise ValueError(f"need a (k, {self.n}) block and its (k, {self.nrhs}) right-hand sides")
        if k > self.rows:
            raise ValueError(f"cannot remove {k} rows from a problem of {self.rows}")
        A = colmajor_empty(self.n, self.n, self.device)
        A.copy_(self.A)
        α, c = self.α.clone(), colmajor_empty(self.n, self.nrhs, self.device)
        c.copy_(self.c)
        drop = torch.zeros_like(self._ss)
        infos = []
        for r0 in range(0, k, self._cap):
            r1 = min(k, r0 + self._cap)
            Z = to_colmajor(A_blk[r0:r1], device=self.device)
            e = to_colmajor(b_blk[r0:r1], device=self.device)
            d = downdate_rows_((A, α), Z, self.handle)
            d.apply_(c, e)
            drop += (e * e).sum(0)
            infos.append(d.info)
        info = torch.cat(infos).cpu() if infos else torch.zeros(0, dtype=torch.int64)
        bad = info.nonzero()
        if len(bad):
            b = int(bad[0, 0])
            raise ValueError(f"removing these rows is impossible: the downdate fails at column {int(info[b])} (rows "
                             f"{b * self._cap}..{min(k, (b + 1) * self._cap) - 1} of the block); were they ever added?")
        self.A, self.α, self.c = A, α, c
        self._ss -= drop
        self.rows -= k
        return self

    @property
    def alpha(self):
        return self.α

    @property
    def R(self) -> torch.Tensor:
        """The n x n triangle R' of every row added so far."""
        return form_r(self.A, self.α)

    def solve(self) -> torch.Tensor:
        """x = R'^{-1} c through backsolve_; neither R nor c is modified."""
        x = colmajor_empty(self.n, self.nrhs, self.device)
        x.copy_(self.c)
        backsolve_(x, self.A, self.α, self.handle)
        return x[:, 0] if self.nrhs == 1 else x

    def residual_norm(self) -> torch.Tensor:
        """||A x - b|| per right-hand side at the least-squares solution, accumulated as the blocks were folded in (and taken out:
        rounding can then take the accumulated sum of squares slightly below 0 when the residual is about 0, so it is clamped)."""
        return self._ss.clamp(min=0).sqrt()


# --------------------------------------------------------------------------------------------
# batched QR of many small problems (torch.geqrf / torch.linalg.lstsq on a batch; cuBLAS geqrfBatched / gelsBatched)
# --------------------------------------------------------------------------------------------
def colmajor_empty_batched(batch: int, m: int, n: int, device="cuda", lda: Optional[int] = None, stride: Optional[int] = None,
                           dtype=torch.float64) -> torch.Tensor:
    """(batch, m, n) tensor whose matrices are column-major: strides (stride, 1, lda), lda default m, stride default lda * n."""
    lda = max(int(lda or m), 1)
    stride = int(stride if stride is not None else lda * max(n, 1))
    if stride < lda * n:
        raise ValueError(f"stride {stride} < lda * n = {lda * n}")
    base = torch.empty(max(batch * stride, 1), dtype=dtype, device=device)
    return base.as_strided((batch, m, n), (stride, 1, lda))


def _batched_args(A: torch.Tensor):
    """(batch, m, n, lda, stride_a) of a (batch, m, n) float64 CUDA tensor of column-major matrices; ValueError otherwise."""
    if not isinstance(A, torch.Tensor) or not A.is_cuda or A.dtype != torch.float64 or A.dim() != 3:
        raise ValueError("A must be a (batch, m, n) float64 CUDA tensor")
    batch, m, n = A.shape
    if m > 1 and A.stride(1) != 1:
        raise ValueError("the matrices of A must be column-major: stride(-2) == 1 (see colmajor_empty_batched)")
    lda = A.stride(2) if n > 1 else max(m, 1)
    if lda < max(m, 1):
        raise ValueError("stride(-1) of A is smaller than the row count")
    if batch > 1 and A.stride(0) < lda * n:
        raise ValueError("stride(0) of A is smaller than stride(-1) * n: the matrices overlap")
    return batch, m, n, lda, A.stride(0)


def _batched_rhs(b: torch.Tensor, batch: int, m: int):
    """(ldb, stride_b, nrhs) of b: (batch, m) or (batch, m, k) float64 on the device, each block column-major."""
    if not isinstance(b, torch.Tensor) or not b.is_cuda or b.dtype != torch.float64 or b.dim() not in (2, 3):
        raise ValueError("b must be a (batch, m) or (batch, m, k) float64 CUDA tensor")
    if b.shape[0] != batch or b.shape[1] != m:
        raise ValueError(f"b must have shape ({batch}, {m}) or ({batch}, {m}, k), not {tuple(b.shape)}")
    nrhs = 1 if b.dim() == 2 else b.shape[2]
    if m > 1 and b.stride(1) != 1:
        raise ValueError("the right-hand sides must be column-major: stride(1) == 1")
    ldb = b.stride(2) if b.dim() == 3 and nrhs > 1 else max(m, 1)
    if ldb < max(m, 1):
        raise ValueError("stride(-1) of b is smaller than the row count")
    if batch > 1 and b.stride(0) < ldb * nrhs:
        raise ValueError("stride(0) of b is smaller than stride(-1) * k: the blocks overlap")
    return ldb, b.stride(0), nrhs


def _check_batch_limit(h: Handle, m: int, n: int) -> None:
    lim = h.get_option("batch_max_elems")
    if n > m:
        raise ValueError(f"the batched QR takes n <= m, not {m} x {n}")
    if m * n > lim:
        raise ValueError(f"{m} x {n} = {m * n} elements exceeds batch_max_elems = {lim}: factor problems this large one at a time with qr_")


class BatchedHouseholderQRStruct:
    """The factorisations of a batch from ``qr_batched_``: ``.A`` (the caller's (batch, m, n) storage, factored in place) and ``.α``
    (``.alpha``, (batch, n)).  Problem i is ``(A[i], α[i])`` in the library's storage format, so every single-problem entry point
    takes it as a factorisation."""

    def __init__(self, A: torch.Tensor, alpha: torch.Tensor, handle: Handle):
        self.A, self.α, self.handle = A, alpha, handle

    @property
    def alpha(self):
        return self.α

    def apply_qt_(self, b: torch.Tensor) -> torch.Tensor:
        return apply_qt_batched_(b, self.A, self.handle)

    def apply_q_(self, b: torch.Tensor) -> torch.Tensor:
        return apply_q_batched_(b, self.A, self.handle)

    def ldiv(self, b, return_residual: bool = False):
        """Least squares min ||A_i x - b_i|| for every problem: ``b`` (batch, m) or (batch, m, k) is left untouched; returns x,
        (batch, n) or (batch, n, k), and with ``return_residual`` also the residual norms ||A_i x - b_i||, (batch,) or (batch, k)."""
        batch, m, n, _, _ = _batched_args(self.A)
        b = torch.as_tensor(b)
        if b.dim() not in (2, 3) or b.shape[0] != batch or b.shape[1] != m:
            raise ValueError(f"b must have shape ({batch}, {m}) or ({batch}, {m}, k)")
        k = 1 if b.dim() == 2 else b.shape[2]
        s = colmajor_empty_batched(batch, m, k, self.A.device)
        s.copy_(b.to(device=self.A.device, dtype=torch.float64).reshape(batch, m, k))
        solve_batched_(s, self.A, self.α, self.handle)
        x = s[:, :n].clone()
        res = torch.linalg.vector_norm(s[:, n:], dim=1)
        if b.dim() == 2:
            x, res = x[..., 0], res[..., 0]
        return (x, res) if return_residual else x


def qr_batched_(A: torch.Tensor, handle: Optional[Handle] = None) -> BatchedHouseholderQRStruct:
    """Factor every matrix of ``A`` ((batch, m, n) float64, column-major matrices: stride(-2) == 1, stride(-1) >= m,
    stride(0) >= stride(-1) * n) in place, in one launch.  n <= m and m * n <= batch_max_elems (196 608); a larger problem raises
    ValueError (qr_ factors it).  Bitwise deterministic per problem, whatever the batch around it."""
    batch, m, n, lda, sa = _batched_args(A)
    h = handle or default_handle(A.device.index)
    _check_batch_limit(h, m, n)
    alpha = torch.empty(batch, n, dtype=torch.float64, device=A.device)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_qr_batched_f64", h.raw, m, n, batch, C.c_void_p(A.data_ptr()), lda, sa, C.c_void_p(alpha.data_ptr()), n,
                  _stream_ptr(A.device))
    return BatchedHouseholderQRStruct(A, alpha, h)


def _apply_batched(fn: str, b: torch.Tensor, A: torch.Tensor, handle: Optional[Handle], alpha: Optional[torch.Tensor] = None):
    batch, m, n, lda, sa = _batched_args(A)
    h = handle or default_handle(A.device.index)
    _check_batch_limit(h, m, n)
    ldb, sb, nrhs = _batched_rhs(b, batch, m)
    args = [h.raw, m, n, batch, C.c_void_p(A.data_ptr()), lda, sa]
    if alpha is not None:
        if alpha.dtype != torch.float64 or alpha.dim() != 2 or tuple(alpha.shape) != (batch, n) or (n > 1 and alpha.stride(1) != 1):
            raise ValueError(f"alpha must be a ({batch}, {n}) float64 tensor with contiguous rows")
        args += [C.c_void_p(alpha.data_ptr()), alpha.stride(0)]
    with torch.cuda.device(A.device):
        _lib.call(fn, *args, C.c_void_p(b.data_ptr()), ldb, sb, nrhs, _stream_ptr(A.device))
    return b


def apply_qt_batched_(b: torch.Tensor, A: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """b_i <- Q_i' b_i for every problem of a batch factored by qr_batched_; ``b`` (batch, m) or (batch, m, k), in place."""
    return _apply_batched("dhqr_apply_qt_batched_f64", b, A, handle)


def apply_q_batched_(b: torch.Tensor, A: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """b_i <- Q_i b_i for every problem of a batch factored by qr_batched_; ``b`` (batch, m) or (batch, m, k), in place."""
    return _apply_batched("dhqr_apply_q_batched_f64", b, A, handle)


def solve_batched_(b: torch.Tensor, A: torch.Tensor, alpha: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """Q'b and the back-substitution in one launch, in place: on return b[:, :n] = x and b[:, n:] = rows n..m-1 of Q'b, whose
    norm is the residual norm.  Returns b."""
    return _apply_batched("dhqr_solve_batched_f64", b, A, handle, alpha)


# --------------------------------------------------------------------------------------------
# rows into and out of many small triangles in one launch, and their back-substitution (DESIGN §2.13)
# --------------------------------------------------------------------------------------------
class BatchedAppendedRows:
    """The reflectors of ``append_rows_batched_``: ``.B`` holds problem i's tails V2 in B[i] (the caller's (batch, k, n) block,
    overwritten) and ``.vtop`` ((batch, n)) their tops, so ``AppendedRows(B[i], vtop[i], handle)`` applies problem i's Q~."""

    def __init__(self, B, vtop, handle: Handle):
        self.B, self.vtop, self.handle = B, vtop, handle


class BatchedDowndatedRows(BatchedAppendedRows):
    """The hyperbolic reflectors of ``downdate_rows_batched_`` (``.B``, ``.vtop``) and ``.info``, a (batch,) int64 CUDA tensor: 0, or
    the 1-based column at which problem i's removal proved impossible.  Reading it synchronises with the device."""

    def __init__(self, B, vtop, info, handle: Handle):
        super().__init__(B, vtop, handle)
        self.info = info


def _vector_batch(x: torch.Tensor, batch: int, n: int, what: str) -> int:
    """stride(0) of a (batch, n) float64 CUDA tensor with contiguous rows."""
    if (not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.float64 or tuple(x.shape) != (batch, n)
            or (n > 1 and x.stride(1) != 1)):
        raise ValueError(f"{what} must be a ({batch}, {n}) float64 CUDA tensor with contiguous rows")
    return x.stride(0)


def _check_update_limit(h: Handle, n: int, k: int, nrhs: int) -> None:
    cols, lim = h.get_option("batch_update_max_cols"), h.get_option("batch_max_elems")
    if n + nrhs > cols:
        raise ValueError(f"n + nrhs = {n + nrhs} exceeds batch_update_max_cols = {cols}")
    if k * (n + nrhs) > lim:
        raise ValueError(f"k * (n + nrhs) = {k * (n + nrhs)} exceeds batch_max_elems = {lim}: split the block "
                         "(BatchedStreamingLeastSquares does)")


def _tp_batched(fn: str, R: torch.Tensor, alpha: torch.Tensor, B: torch.Tensor, c, e, handle: Optional[Handle], hyp: bool):
    batch, m, n, ldr, sr = _batched_args(R)
    if m < n:
        raise ValueError(f"R must hold (batch, m, n) matrices with m >= n, not {tuple(R.shape)}")
    sal = _vector_batch(alpha, batch, n, "alpha")
    bb, k, nb, ldb, sb = _batched_args(B)
    if bb != batch or nb != n:
        raise ValueError(f"B must have shape ({batch}, k, {n}), not {tuple(B.shape)}")
    if (c is None) != (e is None):
        raise ValueError("pass both c and e, or neither")
    nrhs, rhs = 0, [None, 0, 0, None, 0, 0]
    if c is not None:
        ldc, sc, nrhs = _batched_rhs(c, batch, n)
        lde, se, nrhs_e = _batched_rhs(e, batch, k)
        if nrhs != nrhs_e:
            raise ValueError("c and e must have the same number of right-hand sides")
        rhs = [C.c_void_p(c.data_ptr()), ldc, sc, C.c_void_p(e.data_ptr()), lde, se]
    h = handle or default_handle(R.device.index)
    _check_update_limit(h, n, k, nrhs)
    vtop = torch.zeros(batch, n, dtype=torch.float64, device=R.device)
    info = torch.zeros(batch, dtype=torch.int64, device=R.device) if hyp else None
    args = [h.raw, n, k, batch, C.c_void_p(R.data_ptr()), ldr, sr, C.c_void_p(alpha.data_ptr()), sal, C.c_void_p(B.data_ptr()), ldb, sb,
            C.c_void_p(vtop.data_ptr()), n, *rhs, nrhs]
    if hyp:
        args.append(C.c_void_p(info.data_ptr()))
    with torch.cuda.device(R.device):
        _lib.call(fn, *args, _stream_ptr(R.device))
    return (BatchedDowndatedRows(B, vtop, info, h) if hyp else BatchedAppendedRows(B, vtop, h))


def append_rows_batched_(R: torch.Tensor, alpha: torch.Tensor, B: torch.Tensor, c: Optional[torch.Tensor] = None,
                         e: Optional[torch.Tensor] = None, handle: Optional[Handle] = None) -> BatchedAppendedRows:
    """Fold the k new rows ``B[i]`` into the triangle of every problem i, in one launch: ``R`` (batch, m, n) column-major matrices
    with m >= n whose strict upper n x n triangles hold R (a qr_batched_ factorisation works; the diagonal and lower part are never
    touched), ``alpha`` (batch, n) its diagonal, ``B`` (batch, k, n) column-major, overwritten with the reflector tails.  With ``c``
    ((batch, n) or (batch, n, nrhs)) and ``e`` ((batch, k) or (batch, k, nrhs)), [c; e] <- Q~'[c; e] in the same launch.  n + nrhs <=
    batch_update_max_cols and k (n + nrhs) <= batch_max_elems.  Stream-ordered, no synchronisation."""
    return _tp_batched("dhqr_qr_append_batched_f64", R, alpha, B, c, e, handle, False)


def downdate_rows_batched_(R: torch.Tensor, alpha: torch.Tensor, Z: torch.Tensor, c: Optional[torch.Tensor] = None,
                           e: Optional[torch.Tensor] = None, handle: Optional[Handle] = None) -> BatchedDowndatedRows:
    """Remove the k rows ``Z[i]`` from the triangle of every problem i, in one launch (operands as for append_rows_batched_; with
    ``c`` and ``e``, [c; e] <- Theta [c; e]).  ``.info[i]`` is 0, or the 1-based column at which problem i's removal proved
    impossible; from that column on its alpha is NaN.  Stream-ordered, no synchronisation."""
    return _tp_batched("dhqr_qr_downdate_batched_f64", R, alpha, Z, c, e, handle, True)


def backsolve_batched_(b: torch.Tensor, R: torch.Tensor, alpha: torch.Tensor, handle: Optional[Handle] = None) -> torch.Tensor:
    """b_i[0:n] <- R_i^{-1} b_i[0:n] for every problem, in place, in one launch: ``R`` and ``alpha`` as for append_rows_batched_
    (only R's strict upper triangle and alpha are read), ``b`` (batch, m) or (batch, m, k) with m >= n, column-major blocks; rows
    n..m-1 are left alone.  n <= batch_update_max_cols.  Returns b."""
    batch, m, n, ldr, sr = _batched_args(R)
    if m < n:
        raise ValueError(f"R must hold (batch, m, n) matrices with m >= n, not {tuple(R.shape)}")
    sal = _vector_batch(alpha, batch, n, "alpha")
    if not isinstance(b, torch.Tensor) or b.dim() not in (2, 3) or b.shape[0] != batch or b.shape[1] < n:
        raise ValueError(f"b must be a ({batch}, m) or ({batch}, m, k) tensor with m >= {n}")
    ldb, sb, nrhs = _batched_rhs(b, batch, b.shape[1])
    h = handle or default_handle(R.device.index)
    if n > h.get_option("batch_update_max_cols"):
        raise ValueError(f"n = {n} exceeds batch_update_max_cols = {h.get_option('batch_update_max_cols')}")
    with torch.cuda.device(R.device):
        _lib.call("dhqr_backsolve_batched_f64", h.raw, n, batch, C.c_void_p(R.data_ptr()), ldr, sr, C.c_void_p(alpha.data_ptr()), sal,
                  C.c_void_p(b.data_ptr()), ldb, sb, nrhs, _stream_ptr(R.device))
    return b


class BatchedStreamingLeastSquares:
    """min ||A_i x_i - b_i|| for ``batch`` independent problems of n unknowns, fed block by block: ``add`` folds the rows of a
    (batch, k, n) block into every triangle (from R = 0) and their right-hand sides into c = (Q'b)[0:n]; ``remove`` takes rows out
    again, so add-newest / remove-oldest / solve keeps a rolling window per problem at O(k n^2) per slide::

        ls = BatchedStreamingLeastSquares(batch, n)
        for A_blk, b_blk in blocks:            # (batch, k, n), (batch, k)
            ls.add(A_blk, b_blk)
            window.append((A_blk, b_blk))
            if len(window) > w:
                ls.remove(*window.pop(0))
            x = ls.solve()                     # (batch, n)

    Each of ``add``, ``remove`` and ``solve`` is one library launch (plus torch copies) while k (n + nrhs) <= batch_max_elems;
    larger blocks are split.  Nothing synchronises: ``remove`` returns the (batch,) int64 device tensor of its downdates' status,
    0 where the rows came out, and a problem whose removal failed (the rows were never added, or the remaining rows are
    rank-deficient) keeps its previous R, alpha, c, sum of squares and row count."""

    def __init__(self, batch: int, n: int, nrhs: int = 1, device=0, handle: Optional[Handle] = None):
        self.batch, self.n, self.nrhs = int(batch), int(n), int(nrhs)
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        self.handle = handle or default_handle(self.device.index)
        cols = self.handle.get_option("batch_update_max_cols")
        if self.n < 1 or self.nrhs < 1 or self.n + self.nrhs > cols:
            raise ValueError(f"need n >= 1, nrhs >= 1 and n + nrhs <= batch_update_max_cols = {cols}")
        self._cap = self.handle.get_option("batch_max_elems") // (self.n + self.nrhs)
        self.A = colmajor_empty_batched(self.batch, self.n, self.n, self.device)
        self.A.zero_()
        self.α = torch.zeros(self.batch, self.n, dtype=torch.float64, device=self.device)
        self.c = colmajor_empty_batched(self.batch, self.n, self.nrhs, self.device)
        self.c.zero_()
        self._ss = torch.zeros(self.batch, self.nrhs, dtype=torch.float64, device=self.device)
        self.rows = torch.zeros(self.batch, dtype=torch.int64, device=self.device)

    def _copy(self, x: torch.Tensor) -> torch.Tensor:
        y = colmajor_empty_batched(x.shape[0], x.shape[1], x.shape[2], self.device)
        return y.copy_(x)

    def _blocks(self, A_blk, b_blk):
        """(k, [(B, e), ...]): column-major copies of the block in pieces of at most k (n + nrhs) <= batch_max_elems rows."""
        A_blk = torch.as_tensor(A_blk, device=self.device, dtype=torch.float64)
        b_blk = torch.as_tensor(b_blk, device=self.device, dtype=torch.float64)
        if b_blk.dim() == 2:
            b_blk = b_blk[..., None]
        if A_blk.dim() != 3 or A_blk.shape[0] != self.batch or A_blk.shape[2] != self.n:
            raise ValueError(f"need a ({self.batch}, k, {self.n}) block, not {tuple(A_blk.shape)}")
        k = A_blk.shape[1]
        if tuple(b_blk.shape) != (self.batch, k, self.nrhs):
            raise ValueError(f"need ({self.batch}, {k}) or ({self.batch}, {k}, {self.nrhs}) right-hand sides")
        return k, [(self._copy(A_blk[:, r0:r0 + self._cap]), self._copy(b_blk[:, r0:r0 + self._cap])) for r0 in range(0, k, self._cap)]

    def add(self, A_blk, b_blk) -> "BatchedStreamingLeastSquares":
        """Fold rows ``A_blk`` (batch, k, n) with right-hand sides ``b_blk`` ((batch, k) or (batch, k, nrhs)) into every problem."""
        k, blocks = self._blocks(A_blk, b_blk)
        for B, e in blocks:
            append_rows_batched_(self.A, self.α, B, self.c, e, self.handle)
            self._ss += (e * e).sum(1)
        self.rows += k
        return self

    def remove(self, A_blk, b_blk) -> torch.Tensor:
        """Take rows ``A_blk`` (batch, k, n) with right-hand sides ``b_blk`` out of every problem again: they must be rows that were
        added.  R, alpha and c are downdated as copies, and each problem takes its copy only where every block's removal succeeded.
        Returns the (batch,) int64 status on the device (0, or the 1-based column at which the first failing block showed the
        removal impossible); nothing synchronises."""
        k, blocks = self._blocks(A_blk, b_blk)
        A, α, c = self._copy(self.A), self.α.clone(), self._copy(self.c)
        drop = torch.zeros_like(self._ss)
        info = torch.zeros(self.batch, dtype=torch.int64, device=self.device)
        for Z, e in blocks:
            d = downdate_rows_batched_(A, α, Z, c, e, self.handle)
            drop += (e * e).sum(1)
            info = torch.where(info != 0, info, d.info)
        ok = info == 0
        self.A.copy_(torch.where(ok[:, None, None], A, self.A))
        self.α.copy_(torch.where(ok[:, None], α, self.α))
        self.c.copy_(torch.where(ok[:, None, None], c, self.c))
        self._ss -= torch.where(ok[:, None], drop, torch.zeros_like(drop))
        self.rows -= torch.where(ok, k, 0)
        return info

    @property
    def alpha(self):
        return self.α

    @property
    def R(self) -> torch.Tensor:
        """(batch, n, n): the triangle R' of every problem's rows."""
        return torch.triu(self.A, 1) + torch.diag_embed(self.α)

    def solve(self) -> torch.Tensor:
        """x_i = R_i'^{-1} c_i for every problem through backsolve_batched_: (batch, n), or (batch, n, nrhs); R and c are kept."""
        x = self._copy(self.c)
        backsolve_batched_(x, self.A, self.α, self.handle)
        return x[..., 0] if self.nrhs == 1 else x

    def residual_norm(self) -> torch.Tensor:
        """||A_i x_i - b_i|| per problem (and right-hand side) at the least-squares solution, accumulated as blocks were added and
        removed, the sum of squares clamped at 0 against rounding: (batch,), or (batch, nrhs)."""
        r = self._ss.clamp(min=0).sqrt()
        return r[:, 0] if self.nrhs == 1 else r
