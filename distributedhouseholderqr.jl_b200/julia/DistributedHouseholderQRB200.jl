# DistributedHouseholderQRB200.jl — drop-in for DistributedHouseholderQR.qr! / \ on H100 GPUs.
#
# UNEXECUTED in this repository's CI image (no Julia there); it documents the reference-side binding a
# maintainer adds.  Every method names the reference method it replaces
# (S:n = src/DistributedHouseholderQR.jl:n of jwscook/DistributedHouseholderQR.jl).
#
# One Julia worker per GPU (mirrors `procs(A)` of S:116): the DArray's localpart on each worker is a
# CuMatrix{Float64}; libdhqr.so does the arithmetic and the NVLink exchange (NCCL), Distributed.jl only
# ships the 128-byte NCCL unique id and triggers the SPMD call.
module DistributedHouseholderQRB200

using CUDA, Distributed, DistributedArrays, LinearAlgebra

const libdhqr = get(ENV, "DHQR_LIB", "libdhqr.so")

struct DhqrError <: Exception
    fn::Symbol
    code::Cint
    msg::String
end
check(fn::Symbol, rc::Cint) = rc == 0 ? nothing :
    throw(DhqrError(fn, rc, unsafe_string(ccall((:dhqr_last_error, libdhqr), Cstring, ()))))

mutable struct Handle
    ptr::Ptr{Cvoid}
end
function Handle(device::Integer = CUDA.deviceid(CUDA.device()))
    r = Ref{Ptr{Cvoid}}(C_NULL)
    check(:dhqr_create, ccall((:dhqr_create, libdhqr), Cint, (Ref{Ptr{Cvoid}}, Cint), r, device))
    h = Handle(r[]); finalizer(destroy!, h); h
end
function Handle(device::Integer, uid::Vector{UInt8}, rank::Integer, nranks::Integer)
    r = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve uid check(:dhqr_create_dist, ccall((:dhqr_create_dist, libdhqr), Cint,
        (Ref{Ptr{Cvoid}}, Cint, Ptr{UInt8}, Cint, Cint), r, device, pointer(uid), rank, nranks))
    h = Handle(r[]); finalizer(destroy!, h); h
end
destroy!(h::Handle) = (h.ptr == C_NULL || ccall((:dhqr_destroy, libdhqr), Cint, (Ptr{Cvoid},), h.ptr); h.ptr = C_NULL)
nccl_unique_id() = (u = zeros(UInt8, 128);
    check(:dhqr_nccl_unique_id, ccall((:dhqr_nccl_unique_id, libdhqr), Cint, (Ptr{UInt8},), u)); u)

const HANDLE = Ref{Union{Nothing,Handle}}(nothing)
handle() = something(HANDLE[], (HANDLE[] = Handle(); HANDLE[]))

"One-time setup on the master: build the NCCL communicator over workers() (one GPU each)."
function init_distributed!(pids = workers())
    uid = remotecall_fetch(nccl_unique_id, pids[1])                                  # rank 0 mints the id
    @sync for (r, p) in enumerate(pids)
        @spawnat p (CUDA.device!(r - 1); HANDLE[] = Handle(r - 1, uid, r - 1, length(pids)))
    end
end

# S:296-309
struct DistributedHouseholderQRStruct{T1, T2}
    A::T1
    α::T2
end

stream_ptr() = reinterpret(Ptr{Cvoid}, CUDA.stream().handle)

# ---- qr!(A::CuMatrix)  replaces S:311-315 with householder!(A, α) S:113 / _householder! S:122-148 ----
function householder!(A::CuMatrix{Float64}, α::CuVector{Float64}; nb::Integer = 0)
    m, n = size(A)
    GC.@preserve A α check(:dhqr_qr_f64, ccall((:dhqr_qr_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, 0, n, pointer(A), stride(A, 2), pointer(α), nb, stream_ptr()))
    (A, α)
end
function qr!(A::CuMatrix{Float64}; nb::Integer = 0)
    H = DistributedHouseholderQRStruct(A, CUDA.zeros(Float64, size(A, 2)))            # S:306-309
    householder!(H.A, H.α; nb)                                                          # S:313
    return H
end

# ---- qr!(A::Matrix) — a host-resident matrix (S:311 takes any AbstractMatrix): dhqr_qr_host_f64 uploads, factors and downloads
# inside one call.  With page-locked memory (`pin = true`: CUDA.pin registers the array in place) the call is a pipeline - chunked
# upload, one factorisation on a growing window, finished panels stream back (DESIGN 2.5); with pageable memory it is still correct.
function qr!(A::Matrix{Float64}; nb::Integer = 0, pin::Bool = true)
    m, n = size(A)
    α = Vector{Float64}(undef, n)
    pin && (CUDA.pin(A); CUDA.pin(α))
    GC.@preserve A α check(:dhqr_qr_host_f64, ccall((:dhqr_qr_host_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Ptr{Float64}, Int64, Ptr{Float64}, Cint),
        handle().ptr, m, n, pointer(A), stride(A, 2), pointer(α), nb))
    return DistributedHouseholderQRStruct(A, α)                                        # H.A === A (S:314)
end
# H \ b for that host-resident factorisation (S:317-321): b untouched, x is a new vector
function LinearAlgebra.:(\)(H::DistributedHouseholderQRStruct{<:Matrix{Float64}}, b0::AbstractVector)
    m, n = size(H.A)
    length(b0) == m || throw(DimensionMismatch("b must have length $m"))
    b = Vector{Float64}(b0)
    x = Vector{Float64}(undef, n)
    GC.@preserve H b x check(:dhqr_ldiv_host_f64, ccall((:dhqr_ldiv_host_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Ptr{Float64}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
        handle().ptr, m, n, pointer(H.A), stride(H.A, 2), pointer(H.α), pointer(b), pointer(x)))
    return x
end

# ---- qr!(A::DArray) replaces S:115-119: SPMD call on every owner instead of the sequential owner loop ----
function local_qr!(A::DArray, n::Int, nb::Integer)
    Al = localpart(A)::CuMatrix{Float64}
    col0 = first(DistributedArrays.localindices(A)[2]) - 1                              # Δj of S:34
    α = CUDA.zeros(Float64, n)
    m = size(A, 1)
    GC.@preserve Al α check(:dhqr_qr_f64, ccall((:dhqr_qr_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, col0, size(Al, 2), pointer(Al), stride(Al, 2), pointer(α), nb, stream_ptr()))
    CUDA.synchronize()
    return Array(α)                                                                      # replicated: every rank holds all of α
end
function qr!(A::DArray; nb::Integer = 0)
    n = size(A, 2)
    αs = asyncmap(p -> remotecall_fetch(local_qr!, p, A, n, nb), procs(A))              # all owners at once (SPMD)
    return DistributedHouseholderQRStruct(A, αs[1])                                      # S:301-304 (α was a SharedArray)
end

# ---- H \ b replaces S:317-321 (solve_householder! S:284-294) ----
function LinearAlgebra.:(\)(H::DistributedHouseholderQRStruct{<:CuMatrix}, b::AbstractVector)
    A = H.A; m, n = size(A)
    s = CuVector{Float64}(b)                                                             # S:318: b itself is never touched
    GC.@preserve A s check(:dhqr_solve_f64, ccall((:dhqr_solve_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, 0, n, pointer(A), stride(A, 2), pointer(H.α), pointer(s), m, 1, stream_ptr()))
    return Array(s[1:n])                                                                 # S:320
end
function local_solve(A::DArray, α::Vector{Float64}, b::Vector{Float64})
    Al = localpart(A)::CuMatrix{Float64}
    col0 = first(DistributedArrays.localindices(A)[2]) - 1
    m, n = size(A)
    s = CuVector{Float64}(b); dα = CuVector{Float64}(α)
    GC.@preserve Al s dα check(:dhqr_solve_f64, ccall((:dhqr_solve_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, col0, size(Al, 2), pointer(Al), stride(Al, 2), pointer(dα), pointer(s), m, 1, stream_ptr()))
    return Array(s[1:n])
end
function LinearAlgebra.:(\)(H::DistributedHouseholderQRStruct{<:DArray}, b::AbstractVector)
    xs = asyncmap(p -> remotecall_fetch(local_solve, p, H.A, H.α, Vector{Float64}(b)), procs(H.A))
    return xs[1]
end

# ---- ComplexF64 (the reference's second element type, test/runtests.jl:43; S:9, S:51-59, S:162-196), single GPU ----
function qr!(A::CuMatrix{ComplexF64})
    m, n = size(A)
    α = CUDA.zeros(ComplexF64, n)
    GC.@preserve A α check(:dhqr_qr_c64, ccall((:dhqr_qr_c64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{ComplexF64}, Int64, CuPtr{ComplexF64}, Ptr{Cvoid}),
        handle().ptr, m, n, 0, n, pointer(A), stride(A, 2), pointer(α), stream_ptr()))
    return DistributedHouseholderQRStruct(A, α)
end
function LinearAlgebra.:(\)(H::DistributedHouseholderQRStruct{<:CuMatrix{ComplexF64}}, b::AbstractVector)
    A = H.A; m, n = size(A)
    s = CuVector{ComplexF64}(b)                                                          # S:318
    GC.@preserve A s check(:dhqr_solve_c64, ccall((:dhqr_solve_c64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{ComplexF64}, Int64, CuPtr{ComplexF64}, CuPtr{ComplexF64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, 0, n, pointer(A), stride(A, 2), pointer(H.α), pointer(s), m, 1, stream_ptr()))
    return Array(s[1:n])                                                                 # S:320
end

# ---- Q'b and Q b as operators (not in the reference, which never forms Q) ----
function apply_qt!(b::CuVecOrMat{Float64}, A::CuMatrix{Float64})
    m, n = size(A)
    GC.@preserve A b check(:dhqr_apply_qt_f64, ccall((:dhqr_apply_qt_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, 0, n, pointer(A), stride(A, 2), pointer(b), max(stride(b, 2), m), size(b, 2), stream_ptr()))
    return b
end
function apply_q!(b::CuVecOrMat{Float64}, A::CuMatrix{Float64})
    m, n = size(A)
    GC.@preserve A b check(:dhqr_apply_q_f64, ccall((:dhqr_apply_q_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, 0, n, pointer(A), stride(A, 2), pointer(b), max(stride(b, 2), m), size(b, 2), stream_ptr()))
    return b
end

# ---- new rows into a factorisation (LAPACK dtpqrt / dtpmqrt; not in the reference), single GPU, DESIGN §2.10 ----
# [R; B] = Q~ [R'; 0]: R' replaces R's strict upper triangle in A and α, B becomes the reflector tails, vtop their tops.
struct AppendedRows
    B::CuMatrix{Float64}
    vtop::CuVector{Float64}
end
function append_rows!(H::DistributedHouseholderQRStruct{<:CuMatrix{Float64}}, B::CuMatrix{Float64})
    k, n = size(B)
    A = H.A
    vtop = CUDA.zeros(Float64, n)
    GC.@preserve A B vtop check(:dhqr_qr_append_f64, ccall((:dhqr_qr_append_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, CuPtr{Float64}, Ptr{Cvoid}),
        handle().ptr, n, k, pointer(A), stride(A, 2), pointer(H.α), pointer(B), max(stride(B, 2), k), pointer(vtop), stream_ptr()))
    return AppendedRows(B, vtop)
end
function apply_qt!(c::CuVecOrMat{Float64}, e::CuVecOrMat{Float64}, T::AppendedRows)
    k, n = size(T.B)
    GC.@preserve T c e check(:dhqr_apply_qt_append_f64, ccall((:dhqr_apply_qt_append_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Cint,
         Ptr{Cvoid}),
        handle().ptr, n, k, pointer(T.B), max(stride(T.B, 2), k), pointer(T.vtop), pointer(c), max(stride(c, 2), n), pointer(e),
        max(stride(e, 2), k), size(c, 2), stream_ptr()))
    return c, e
end
# ---- rows out of a factorisation (LINPACK dchdd; not in the reference), single GPU, DESIGN §2.11 ----
# Θ [R; Z] = [R'; 0] with R'ᵀR' = RᵀR − ZᵀZ: R' replaces R's strict upper triangle in A and α, Z becomes the hyperbolic reflector
# tails, vtop their tops; info (on the device) is 0, or the 1-based column at which the removal proved impossible.
struct DowndatedRows
    B::CuMatrix{Float64}
    vtop::CuVector{Float64}
    info::CuVector{Int64}
end
function downdate_rows!(H::DistributedHouseholderQRStruct{<:CuMatrix{Float64}}, Z::CuMatrix{Float64})
    k, n = size(Z)
    A = H.A
    vtop = CUDA.zeros(Float64, n)
    info = CUDA.zeros(Int64, 1)
    GC.@preserve A Z vtop info check(:dhqr_qr_downdate_f64, ccall((:dhqr_qr_downdate_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Int64},
         Ptr{Cvoid}),
        handle().ptr, n, k, pointer(A), stride(A, 2), pointer(H.α), pointer(Z), max(stride(Z, 2), k), pointer(vtop), pointer(info),
        stream_ptr()))
    return DowndatedRows(Z, vtop, info)
end
# [c; e] <- Θ [c; e]: c = (Qᵀb)[1:n] and e the removed rows' right-hand sides become c' (x' = R' \ c') and e'.
function apply!(c::CuVecOrMat{Float64}, e::CuVecOrMat{Float64}, T::DowndatedRows)
    k, n = size(T.B)
    GC.@preserve T c e check(:dhqr_apply_downdate_f64, ccall((:dhqr_apply_downdate_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Cint,
         Ptr{Cvoid}),
        handle().ptr, n, k, pointer(T.B), max(stride(T.B, 2), k), pointer(T.vtop), pointer(c), max(stride(c, 2), n), pointer(e),
        max(stride(e, 2), k), size(c, 2), stream_ptr()))
    return c, e
end
# ---- many small problems in one launch (cuBLAS geqrfBatched / gelsBatched; not in the reference), single GPU, DESIGN §2.12 ----
# A[:, :, i] (m x n, n <= m, m n <= batch_max_elems) is factored in place for every i; α[:, i] receives diag(R).
function qr_batched!(A::CuArray{Float64,3})
    m, n, batch = size(A)
    α = CUDA.zeros(Float64, n, batch)
    GC.@preserve A α check(:dhqr_qr_batched_f64, ccall((:dhqr_qr_batched_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, Ptr{Cvoid}),
        handle().ptr, m, n, batch, pointer(A), max(stride(A, 2), m), stride(A, 3), pointer(α), n, stream_ptr()))
    return A, α
end
# x[:, :, i] = A_i \ b[:, :, i] (least squares) from qr_batched!'s (A, α); b (m x k x batch) is left untouched.
function ldiv_batched(A::CuArray{Float64,3}, α::CuMatrix{Float64}, b::CuArray{Float64,3})
    m, n, batch = size(A)
    s = copy(b)
    GC.@preserve A α s check(:dhqr_solve_batched_f64, ccall((:dhqr_solve_batched_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Int64, Cint,
         Ptr{Cvoid}),
        handle().ptr, m, n, batch, pointer(A), max(stride(A, 2), m), stride(A, 3), pointer(α), n, pointer(s), max(stride(s, 2), m),
        stride(s, 3), size(s, 2), stream_ptr()))
    return s[1:n, :, :]
end
# ---- rows into and out of many small triangles in one launch (not in the reference), single GPU, DESIGN §2.13 ----
# Problem i: R = triu(R[1:n, 1:n, i], 1) + diag(α[:, i]) (a qr_batched! factorisation works), the k x n block B[:, :, i]
# (overwritten with the reflector tails), [c; e] = [c[:, :, i]; e[:, :, i]] transformed in the same launch (nothing: pass c and e
# with size(c, 2) == 0).  n + nrhs <= batch_update_max_cols and k (n + nrhs) <= batch_max_elems.  Returns vtop (n x batch), and
# for the downdate also info (batch, on the device): 0, or the 1-based column at which problem i's removal proved impossible.
function _tp_batched!(name::Symbol, R::CuArray{Float64,3}, α::CuMatrix{Float64}, B::CuArray{Float64,3}, c::CuArray{Float64,3},
                      e::CuArray{Float64,3}, info)
    m, n, batch = size(R)
    k = size(B, 1)
    nrhs = size(c, 2)
    vtop = CUDA.zeros(Float64, n, batch)
    ptrs = (handle().ptr, n, k, batch, pointer(R), max(stride(R, 2), m), stride(R, 3), pointer(α), n, pointer(B), max(stride(B, 2), k),
            stride(B, 3), pointer(vtop), n, pointer(c), max(stride(c, 2), n), stride(c, 3), pointer(e), max(stride(e, 2), k), stride(e, 3),
            Cint(nrhs))
    if info === nothing
        GC.@preserve R α B vtop c e check(name, ccall((:dhqr_qr_append_batched_f64, libdhqr), Cint,
            (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Int64,
             CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, Int64, Cint, Ptr{Cvoid}), ptrs..., stream_ptr()))
    else
        GC.@preserve R α B vtop c e info check(name, ccall((:dhqr_qr_downdate_batched_f64, libdhqr), Cint,
            (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Int64,
             CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, Int64, Cint, CuPtr{Int64}, Ptr{Cvoid}),
            ptrs..., pointer(info), stream_ptr()))
    end
    return vtop
end
append_rows_batched!(R, α, B, c, e) = _tp_batched!(:dhqr_qr_append_batched_f64, R, α, B, c, e, nothing)
function downdate_rows_batched!(R, α, Z, c, e)
    info = CUDA.zeros(Int64, size(R, 3))
    vtop = _tp_batched!(:dhqr_qr_downdate_batched_f64, R, α, Z, c, e, info)
    return vtop, info
end
# b[1:n, :, i] <- R_i \ b[1:n, :, i] for every problem (only R's strict upper triangle and α are read).
function backsolve_batched!(b::CuArray{Float64,3}, R::CuArray{Float64,3}, α::CuMatrix{Float64})
    m, n, batch = size(R)
    GC.@preserve R α b check(:dhqr_backsolve_batched_f64, ccall((:dhqr_backsolve_batched_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Float64}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, Int64, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, n, batch, pointer(R), max(stride(R, 2), m), stride(R, 3), pointer(α), n, pointer(b), max(stride(b, 2), size(b, 1)),
        stride(b, 3), size(b, 2), stream_ptr()))
    return b
end
# min ||A x - b|| for A fed as row blocks (CuMatrix or Matrix; host blocks are uploaded), from R = 0: x and the residual norm.
function streaming_lstsq(blocks, n::Integer)
    H = DistributedHouseholderQRStruct(CUDA.zeros(Float64, n, n), CUDA.zeros(Float64, n))
    c = CUDA.zeros(Float64, n)
    ss = 0.0
    cap = Ref{Int64}(0)
    check(:dhqr_get_option, ccall((:dhqr_get_option, libdhqr), Cint, (Ptr{Cvoid}, Cstring, Ptr{Int64}), handle().ptr,
                                  "append_max_rows", cap))
    for (Ablk, bblk) in blocks
        for r0 in 1:cap[]:size(Ablk, 1)
            r1 = min(size(Ablk, 1), r0 + cap[] - 1)
            e = CuVector{Float64}(bblk[r0:r1])
            apply_qt!(c, e, append_rows!(H, CuMatrix{Float64}(Ablk[r0:r1, :])))
            ss += sum(abs2, e)
        end
    end
    x = copy(c)
    GC.@preserve H x check(:dhqr_backsolve_f64, ccall((:dhqr_backsolve_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Float64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, n, n, 0, n, pointer(H.A), stride(H.A, 2), pointer(H.α), pointer(x), n, 1, stream_ptr()))
    return Array(x), sqrt(ss)
end

# ---- solves with the adjoint (LAPACK ?gels with TRANS = 'C'; not in the reference), single GPU ----
for (T, fs, sa) in ((Float64, :dhqr_forwardsolve_f64, :dhqr_solve_adj_f64), (ComplexF64, :dhqr_forwardsolve_c64, :dhqr_solve_adj_c64))
    @eval begin
        adj_call(::Val{:forward}, A::CuMatrix{$T}, α::CuVector{$T}, b::CuVecOrMat{$T}) =
            GC.@preserve A α b check($(QuoteNode(fs)), ccall(($(QuoteNode(fs)), libdhqr), Cint,
                (Ptr{Cvoid}, Int64, Int64, CuPtr{$T}, Int64, CuPtr{$T}, CuPtr{$T}, Int64, Cint, Ptr{Cvoid}),
                handle().ptr, size(A, 1), size(A, 2), pointer(A), stride(A, 2), pointer(α), pointer(b), max(stride(b, 2), size(A, 1)),
                size(b, 2), stream_ptr()))
        adj_call(::Val{:solve}, A::CuMatrix{$T}, α::CuVector{$T}, b::CuVecOrMat{$T}) =
            GC.@preserve A α b check($(QuoteNode(sa)), ccall(($(QuoteNode(sa)), libdhqr), Cint,
                (Ptr{Cvoid}, Int64, Int64, CuPtr{$T}, Int64, CuPtr{$T}, CuPtr{$T}, Int64, Cint, Ptr{Cvoid}),
                handle().ptr, size(A, 1), size(A, 2), pointer(A), stride(A, 2), pointer(α), pointer(b), max(stride(b, 2), size(A, 1)),
                size(b, 2), stream_ptr()))
    end
end

# b[1:n, :] <- R^{-H} b[1:n, :] (rows n+1:m untouched); returns that view
function forwardsolve!(b::CuVecOrMat{T}, A::CuMatrix{T}, α::CuVector{T}) where {T<:Union{Float64,ComplexF64}}
    adj_call(Val(:forward), A, α, b)
    return b isa CuVector ? view(b, 1:size(A, 2)) : view(b, 1:size(A, 2), :)
end

# H' \ c: the minimum-norm solution y = Q [R^{-H} c; 0] of A^H y = c (dhqr_solve_adj_*); c (length n, or n x k) is not modified
struct AdjointQR{S<:DistributedHouseholderQRStruct}
    parent::S
end
Base.adjoint(H::DistributedHouseholderQRStruct{<:CuMatrix}) = AdjointQR(H)
function LinearAlgebra.:(\)(Ha::AdjointQR, c::AbstractVecOrMat)
    A = Ha.parent.A; T = eltype(A); m, n = size(A)
    size(c, 1) == n || throw(DimensionMismatch("c must have $n rows"))
    y = CUDA.zeros(T, m, size(c, 2))
    y[1:n, :] .= CuArray{T}(reshape(c, n, :))
    adj_call(Val(:solve), A, Ha.parent.α, y)
    return c isa AbstractVector ? vec(y) : y
end

# ---- QR with column pivoting (LAPACK dgeqp3 / zgeqp3; not in the reference), Float64 and ComplexF64, single GPU ----
# A[:, p] = Q R: (A, α) is the factorisation of A[:, p] in the storage format above; p is 1-based here, 0-based on the device
struct PivotedHouseholderQRStruct{T1, T2, T3}
    A::T1
    α::T2
    jpvt::T3          # CuVector{Int64}, 0-based
end
Base.getproperty(H::PivotedHouseholderQRStruct, s::Symbol) = s === :p ? Array(getfield(H, :jpvt)) .+ 1 : getfield(H, s)
# numerical rank: the first k with |α_k| <= rtol |α_1| (reads α: synchronises)
function LinearAlgebra.rank(H::PivotedHouseholderQRStruct; rtol::Real = max(size(H.A)...) * eps(Float64))
    a = abs.(Array(H.α))
    isempty(a) && return 0
    k = findfirst(x -> !(x > rtol * a[1]), a)
    return k === nothing ? length(a) : k - 1
end

# ---- complete orthogonal decomposition on the pivoted QR (DESIGN §2.8, §2.9), single GPU ----
# A P ~ Q1 [U^H 0] Z^H at r = rank(H; rtol): (F, γ) is the factorisation R_r^H = Z [U; 0] in the storage format above.  Its \ is the
# minimum-norm solution, the answer the stdlib's qr(A, ColumnNorm()) \ b gives (up to how the rank is picked); \ on the pivoted
# struct itself stays the basic solution.
struct CompleteOrthogonalStruct{T1, T2, T3}
    qrcp::T1
    F::T2
    γ::T3
    rank::Int
end

for (T, qp, sq, cd, sc) in ((Float64, :dhqr_qrcp_f64, :dhqr_solve_qrcp_f64, :dhqr_cod_f64, :dhqr_solve_cod_f64),
                            (ComplexF64, :dhqr_qrcp_c64, :dhqr_solve_qrcp_c64, :dhqr_cod_c64, :dhqr_solve_cod_c64))
    @eval begin
        function qr!(A::CuMatrix{$T}, ::ColumnNorm)
            m, n = size(A)
            α = CUDA.zeros($T, n); jpvt = CUDA.zeros(Int64, n)
            GC.@preserve A α jpvt check($(QuoteNode(qp)), ccall(($(QuoteNode(qp)), libdhqr), Cint,
                (Ptr{Cvoid}, Int64, Int64, CuPtr{$T}, Int64, CuPtr{$T}, CuPtr{Int64}, Ptr{Cvoid}),
                handle().ptr, m, n, pointer(A), stride(A, 2), pointer(α), pointer(jpvt), stream_ptr()))
            return PivotedHouseholderQRStruct(A, α, jpvt)
        end
        # H \ b: the basic solution x = P [R11^{-1} (Q^H b)[1:r]; 0] at r = rank(H; rtol); b is not modified
        function LinearAlgebra.ldiv!(x::AbstractVector, H::PivotedHouseholderQRStruct{<:CuMatrix{$T}}, b::AbstractVector;
                                     rtol::Real = max(size(H.A)...) * eps(Float64))
            A = H.A; m, n = size(A)
            r = rank(H; rtol)
            s = CuVector{$T}(b)
            GC.@preserve A s check($(QuoteNode(sq)), ccall(($(QuoteNode(sq)), libdhqr), Cint,
                (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{$T}, Int64, CuPtr{$T}, CuPtr{Int64}, CuPtr{$T}, Int64, Cint, Ptr{Cvoid}),
                handle().ptr, m, n, r, pointer(A), stride(A, 2), pointer(H.α), pointer(H.jpvt), pointer(s), m, 1, stream_ptr()))
            copyto!(x, Array(s[1:n]))
            return x
        end
        LinearAlgebra.:(\)(H::PivotedHouseholderQRStruct{<:CuMatrix{$T}}, b::AbstractVector) =
            ldiv!(Vector{$T}(undef, size(H.A, 2)), H, b)
        function complete_orthogonal(H::PivotedHouseholderQRStruct{<:CuMatrix{$T}}; rtol::Real = max(size(H.A)...) * eps(Float64))
            A = H.A; m, n = size(A)
            r = rank(H; rtol)
            F = CUDA.zeros($T, n, r); γ = CUDA.zeros($T, r)
            GC.@preserve A F γ check($(QuoteNode(cd)), ccall(($(QuoteNode(cd)), libdhqr), Cint,
                (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{$T}, Int64, CuPtr{$T}, CuPtr{$T}, Int64, CuPtr{$T}, Ptr{Cvoid}),
                handle().ptr, m, n, r, pointer(A), stride(A, 2), pointer(H.α), pointer(F), max(n, 1), pointer(γ), stream_ptr()))
            return CompleteOrthogonalStruct(H, F, γ, r)
        end
        function LinearAlgebra.ldiv!(x::AbstractVector, C::CompleteOrthogonalStruct{<:PivotedHouseholderQRStruct{<:CuMatrix{$T}}},
                                     b::AbstractVector)
            A = C.qrcp.A; m, n = size(A)
            s = CuVector{$T}(b)
            GC.@preserve A s check($(QuoteNode(sc)), ccall(($(QuoteNode(sc)), libdhqr), Cint,
                (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{$T}, Int64, CuPtr{Int64}, CuPtr{$T}, Int64, CuPtr{$T}, CuPtr{$T}, Int64,
                 Cint, Ptr{Cvoid}),
                handle().ptr, m, n, C.rank, pointer(A), stride(A, 2), pointer(C.qrcp.jpvt), pointer(C.F), max(n, 1), pointer(C.γ),
                pointer(s), m, 1, stream_ptr()))
            copyto!(x, Array(s[1:n]))
            return x
        end
        LinearAlgebra.:(\)(C::CompleteOrthogonalStruct{<:PivotedHouseholderQRStruct{<:CuMatrix{$T}}}, b::AbstractVector) =
            ldiv!(Vector{$T}(undef, size(C.qrcp.A, 2)), C, b)
    end
end

end # module
