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
        if b.dim() == 1:
            s = b.to(device=loc.device, dtype=loc.dtype).clone()
        else:
            s = to_colmajor(b, device=loc.device)
        solve_qrcp_(s, self.A, self.α, self.p, r, self.handle)
        return s[:loc.shape[1]].clone(), r

    solve = ldiv


def qrcp_(A: torch.Tensor, handle: Optional[Handle] = None) -> PivotedHouseholderQRStruct:
    """A P = Q R with column pivoting (LAPACK dgeqp3; scipy.linalg.qr(pivoting=True)), in place, on a column-major float64 CUDA
    tensor with n <= m.  Single GPU, stream-ordered, no synchronisation."""
    if not isinstance(A, torch.Tensor) or not A.is_cuda:
        raise TypeError("qrcp_ works on a column-major float64 CUDA tensor")
    if A.dtype != torch.float64:
        raise TypeError("qrcp_ is Float64 only")
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    alpha = torch.zeros(n, dtype=torch.float64, device=A.device)
    p = torch.zeros(n, dtype=torch.int64, device=A.device)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_qrcp_f64", h.raw, m, n, C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(p.data_ptr()), _stream_ptr(A.device))
    return PivotedHouseholderQRStruct(A, alpha, p, h)


def solve_qrcp_(b: torch.Tensor, A: torch.Tensor, alpha: torch.Tensor, p: torch.Tensor, rank: int,
                handle: Optional[Handle] = None) -> torch.Tensor:
    """x = P [R11^{-1} (Q'b)[0:rank]; 0], the basic solution at the given rank, from a factorisation made by ``qrcp_``.  ``b``:
    length m, or (m, k) column-major; on return b[0:n] = x (returned as a view) and rows n..m-1 hold rows n..m-1 of
    H_rank ... H_1 b."""
    h = handle or default_handle(A.device.index)
    m, n = A.shape
    if alpha.dtype != torch.float64 or p.dtype != torch.int64:
        raise TypeError("alpha must be float64 and p int64")
    ldb, nrhs = _rhs_args(b, m, A.dtype)
    with torch.cuda.device(A.device):
        _lib.call("dhqr_solve_qrcp_f64", h.raw, m, n, int(rank), C.c_void_p(A.data_ptr()), _lda(A), C.c_void_p(alpha.data_ptr()),
                  C.c_void_p(p.data_ptr()), C.c_void_p(b.data_ptr()), ldb, nrhs, _stream_ptr(A.device))
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
