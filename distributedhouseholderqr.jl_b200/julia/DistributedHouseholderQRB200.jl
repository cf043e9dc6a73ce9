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

# ---- QR with column pivoting (LAPACK dgeqp3; not in the reference), Float64, single GPU ----
# A[:, p] = Q R: (A, α) is the factorisation of A[:, p] in the storage format above; p is 1-based here, 0-based on the device
struct PivotedHouseholderQRStruct{T1, T2, T3}
    A::T1
    α::T2
    jpvt::T3          # CuVector{Int64}, 0-based
end
function qr!(A::CuMatrix{Float64}, ::ColumnNorm)
    m, n = size(A)
    α = CUDA.zeros(Float64, n); jpvt = CUDA.zeros(Int64, n)
    GC.@preserve A α jpvt check(:dhqr_qrcp_f64, ccall((:dhqr_qrcp_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Int64}, Ptr{Cvoid}),
        handle().ptr, m, n, pointer(A), stride(A, 2), pointer(α), pointer(jpvt), stream_ptr()))
    return PivotedHouseholderQRStruct(A, α, jpvt)
end
Base.getproperty(H::PivotedHouseholderQRStruct, s::Symbol) = s === :p ? Array(getfield(H, :jpvt)) .+ 1 : getfield(H, s)
# numerical rank: the first k with |α_k| <= rtol |α_1| (reads α: synchronises)
function LinearAlgebra.rank(H::PivotedHouseholderQRStruct; rtol::Real = max(size(H.A)...) * eps(Float64))
    a = abs.(Array(H.α))
    isempty(a) && return 0
    k = findfirst(x -> !(x > rtol * a[1]), a)
    return k === nothing ? length(a) : k - 1
end
# H \ b: the basic solution x = P [R11^{-1} (Q'b)[1:r]; 0] at r = rank(H; rtol) (dhqr_solve_qrcp_f64); b is not modified
function LinearAlgebra.ldiv!(x::AbstractVector, H::PivotedHouseholderQRStruct, b::AbstractVector; rtol::Real = max(size(H.A)...) * eps(Float64))
    A = H.A; m, n = size(A)
    r = rank(H; rtol)
    s = CuVector{Float64}(b)
    GC.@preserve A s check(:dhqr_solve_qrcp_f64, ccall((:dhqr_solve_qrcp_f64, libdhqr), Cint,
        (Ptr{Cvoid}, Int64, Int64, Int64, CuPtr{Float64}, Int64, CuPtr{Float64}, CuPtr{Int64}, CuPtr{Float64}, Int64, Cint, Ptr{Cvoid}),
        handle().ptr, m, n, r, pointer(A), stride(A, 2), pointer(H.α), pointer(H.jpvt), pointer(s), m, 1, stream_ptr()))
    copyto!(x, Array(s[1:n]))
    return x
end
LinearAlgebra.:(\)(H::PivotedHouseholderQRStruct, b::AbstractVector) = ldiv!(Vector{Float64}(undef, size(H.A, 2)), H, b)

end # module
