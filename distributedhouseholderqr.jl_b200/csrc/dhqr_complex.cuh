// dhqr_complex.cuh — ComplexF64 path (the reference tests both element types, test/runtests.jl:43; S:9, S:51-59, S:162-196).
//
// A complex reflector H = I - v v^H with |v|^2 = 2 acts on the REAL view of a complex column (re, im interleaved, length 2m) as
// the product of two commuting real reflectors: with v_r = [x0, y0, x1, y1, ...] and v_i = i v = [-y0, x0, -y1, x1, ...]
//     Re(v^H c) = v_r . c_r,   Im(v^H c) = v_i . c_r,   c - v s = c_r - (Re s) v_r - (Im s) v_i,   v_r . v_i = 0, |v_r|^2 = |v_i|^2 = 2
// (partialdot S:51-59 and hotloop! S:162-196 written out in reals).  So the trailing update of a panel of kb complex
// reflectors IS the real block-reflector update with V^ = [v1_r, v1_i, v2_r, v2_i, ...] (2 kb real vectors) on the real view of
// the trailing matrix (2m x n, leading dimension 2 lda), T^{-1} = I + striu(V^' V^): the fp64 tensor-pipe GEMM pair of the real
// path is reused as is (this is the 4M real decomposition of the complex rank-k update).  New here: the complex panel
// factorisation (column by column, S:127-135 with alphafactor(::Complex) S:9), the packing of V^ and the conjugating partialdot
// primitive.  The back- and forward-substitution steps (S:256-282) are here too, written once for Float64 and ComplexF64.
#pragma once
#include <type_traits>

#include "dhqr_kernels.cuh"

namespace dhqr {

constexpr int CPW = 64;   // complex panel width: 64 complex reflectors = 128 real vectors

__device__ __forceinline__ double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ double2 cmulc(double2 a, double2 b) {   // conj(a) * b  (S:51-59: re = ar br + ai bi, im = ar bi - ai br)
    return make_double2(a.x * b.x + a.y * b.y, a.x * b.y - a.y * b.x);
}

__device__ __forceinline__ double2 block_sum2(double2 v, double2* red, int tid, int nthreads) {
    v.x = warp_sum(v.x);
    v.y = warp_sum(v.y);
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    double2 t = make_double2(0.0, 0.0);
    for (int w = 0; w < nthreads / 32; ++w) { t.x += red[w].x; t.y += red[w].y; }   // fixed order
    __syncthreads();
    return t;
}

// sin(pi) in Float64 (Julia's sin(pi), numpy's np.sin(np.pi)): written out rather than left to the device sin
constexpr double SIN_PI = 1.2246467991473532e-16;

// alpha = -exp(i angle(x0)) s  (S:9) of the reflector of a complex column with leading entry x0 and norm s, and a0 = |x0| for its
// scale f = 1 / sqrt(s (s + |x0|)).  angle = atan2(im, re) sees the signs of a zero pivot: angle(+0 +- 0i) = +-0 gives
// alpha = -s, angle(-0 +- 0i) = +-pi gives alpha = -s (cos pi, +-sin pi) = s (1, -+1.2246e-16).  Shared by k_house1_c and the
// pivoted factorisation (dhqr_qrcp.cuh), so both write the same storage format.
__device__ __forceinline__ double2 house_alpha(double2 x0, double s, double& a0) {
    a0 = hypot(x0.x, x0.y);
    // -exp(i angle(x0)) = -(x0 / |x0|); exp(i angle(x0)) = (cos, sin) of +-0 or +-pi for a zero x0
    double ux, uy;
    if (a0 > 0.0) {
        ux = x0.x / a0;
        uy = x0.y / a0;
    } else if (!signbit(x0.x)) {
        ux = 1.0;
        uy = x0.y;
    } else {
        ux = -1.0;
        uy = copysign(SIN_PI, x0.y);
    }
    return make_double2(-ux * s, -uy * s);
}

// S:129-135 for one complex column (one CTA): s = |x|, alpha (house_alpha), f = 1 / sqrt(s (s + |x0|)), x0 -= alpha, x *= f
__global__ void __launch_bounds__(1024, 1) k_house1_c(double2* __restrict__ col, int64_t len, double2* __restrict__ alpha) {
    __shared__ double2 red[32];
    __shared__ double sc[3];
    const int tid = threadIdx.x;
    double2 acc = make_double2(0.0, 0.0);
    for (int64_t i = tid; i < len; i += 1024) {
        const double2 x = col[i];
        acc.x += x.x * x.x + x.y * x.y;
    }
    acc = block_sum2(acc, red, tid, 1024);
    if (tid == 0) {
        const double2 x0 = col[0];
        const double s = sqrt(acc.x);
        double a0;
        const double2 al = house_alpha(x0, s, a0);
        *alpha = al;
        sc[0] = al.x;
        sc[1] = al.y;
        sc[2] = 1.0 / sqrt(s * (s + a0));
    }
    __syncthreads();
    const double f = sc[2];
    for (int64_t i = tid; i < len; i += 1024) {
        double2 x = col[i];
        if (i == 0) { x.x -= sc[0]; x.y -= sc[1]; }
        col[i] = make_double2(x.x * f, x.y * f);
    }
}

// S:198-213 inside the panel: columns jj of C (one CTA each): s = v^H a (S:51-59), a -= v s (S:162-196)
__global__ void __launch_bounds__(256) k_apply1_c(const double2* __restrict__ v, int64_t len, double2* __restrict__ C, int64_t ldc,
                                                  int ncols) {
    __shared__ double2 red[8];
    const int tid = threadIdx.x;
    for (int c = blockIdx.x; c < ncols; c += gridDim.x) {
        double2* col = C + (int64_t)c * ldc;
        double2 acc = make_double2(0.0, 0.0);
        for (int64_t i = tid; i < len; i += 256) {
            const double2 t = cmulc(v[i], col[i]);
            acc.x += t.x;
            acc.y += t.y;
        }
        const double2 s = block_sum2(acc, red, tid, 256);
        for (int64_t i = tid; i < len; i += 256) {
            const double2 t = cmul(v[i], s), a = col[i];
            col[i] = make_double2(a.x - t.x, a.y - t.y);
        }
    }
}

// V^ of a complex panel -> packed V buffer.  A: complex panel top-left (pivot row of complex column 0), complex lda;
// packed column 2j = v_j as reals, 2j+1 = i v_j; complex rows above the diagonal of column j and columns >= kb give zeros;
// real window rows [0, vrows), the panel starts at real window row vtop (even).  grid.y = 128 packed columns.
__global__ void k_pack_c(const double2* __restrict__ A, int64_t lda, int64_t mpc, int kb, double* __restrict__ vpk, int64_t vtop,
                         int64_t vrows) {
    const int pc = blockIdx.y, j = pc >> 1, im = pc & 1;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < vrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pr = r - vtop;                  // real row inside the panel
        double val = 0.0;
        if (j < kb && pr >= 0) {
            const int64_t cr = pr >> 1;               // complex row
            if (cr >= j && cr < mpc) {
                const double2 z = A[(int64_t)j * lda + cr];
                val = (pr & 1) ? (im ? z.x : z.y) : (im ? -z.y : z.x);
            }
        }
        vpk[vpk_index(r, pc)] = val;
    }
}

// ---- substitution steps, T = double or double2 ---------------------------------------------------------------------------------
// What the two step kernels below need of their element type, in overloads.  Each double2 helper fixes the order of its two
// component operations, so every instantiation compiles to the kernel it replaces.
template <typename T> __device__ T zero();
template <> __device__ __forceinline__ double zero<double>() { return 0.0; }
template <> __device__ __forceinline__ double2 zero<double2>() { return make_double2(0.0, 0.0); }

// x -= y and x += y for double2 (y by reference: a copy of it would change the generated code)
__device__ __forceinline__ void operator-=(double2& x, const double2& y) { x.x -= y.x; x.y -= y.y; }
__device__ __forceinline__ void operator+=(double2& x, const double2& y) { x.x += y.x; x.y += y.y; }

// a b and conj(a) b
__device__ __forceinline__ double mul(double a, double b) { return a * b; }
__device__ __forceinline__ double2 mul(double2 a, double2 b) { return cmul(a, b); }
__device__ __forceinline__ double conj_mul(double a, double b) { return a * b; }
__device__ __forceinline__ double2 conj_mul(double2 a, double2 b) { return cmulc(a, b); }

// lane i's v in every lane of the warp, and the sum of v over the warp
__device__ __forceinline__ double shfl(double v, int i) { return __shfl_sync(0xffffffffu, v, i); }
__device__ __forceinline__ double2 shfl(const double2& v, int i) {
    const double x = __shfl_sync(0xffffffffu, v.x, i);
    const double y = __shfl_sync(0xffffffffu, v.y, i);
    return make_double2(x, y);
}
__device__ __forceinline__ double2 warp_sum(const double2& v) {
    const double x = warp_sum(v.x);
    const double y = warp_sum(v.y);
    return make_double2(x, y);
}

// lane i's y over *a in every lane of the warp: the pivot step of the back-substitution.  For double2 *a and |*a|^2 (unscaled) come
// before the shuffles.
__device__ __forceinline__ double shfl_div_alpha(double y, int i, const double* a) { return __shfl_sync(0xffffffffu, y, i) / *a; }
__device__ __forceinline__ double2 shfl_div_alpha(const double2& y, int i, const double2* a) {
    const double2 al = *a;
    const double den = al.x * al.x + al.y * al.y;
    const double nx = __shfl_sync(0xffffffffu, y.x, i), ny = __shfl_sync(0xffffffffu, y.y, i);
    return make_double2((nx * al.x + ny * al.y) / den, (ny * al.x - nx * al.y) / den);
}

// n / conj(a) of the forward substitution.  For double2 by Smith's algorithm: the ratio of the smaller to the larger part of a is
// formed first, so neither |a|^2 nor a partial product overflows or underflows when n and a lie many decades apart (columns scaled
// by 10^+-120).  a = 0 gives NaN.
__device__ __forceinline__ double div_conj(double n, double a) { return n / a; }
__device__ __forceinline__ double2 div_conj(double2 n, double2 a) {
    const double p = a.x, q = -a.y;                                          // conj(a) = p + i q
    if (fabs(p) >= fabs(q)) {
        const double r = q / p, d = p + q * r;
        return make_double2((n.x + n.y * r) / d, (n.y - n.x * r) / d);
    }
    const double r = p / q, d = q + p * r;
    return make_double2((n.x * r + n.y) / d, (n.y * r - n.x) / d);
}

// Back-substitution step (S:256-282), column oriented, for R = triu(A, 1) + diag(alpha): solve the bs x bs diagonal block
//   x_blk = R_bb^{-1} y_blk  in every CTA (one warp), then y[0:c0) -= R[0:c0, blk] x_blk on the CTA's slice of rows.  CTA 0
// publishes x_blk.  Ablk points at (row 0, first column of the block) in local storage; c0 is the global index of that column.
constexpr int BS_BLK = 32;
template <typename T>
__global__ void __launch_bounds__(256) k_backsolve_step(const T* __restrict__ Ablk, int64_t lda, const T* __restrict__ alpha,
                                                        T* __restrict__ y, int64_t ldy, int nrhs, T* __restrict__ x, int64_t ldx,
                                                        int64_t c0, int bs) {
    __shared__ T sx[BS_BLK];
    const int tid = threadIdx.x, lane = tid & 31;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        T* yr = y + (int64_t)rhs * ldy;
        if (tid < 32) {
            T yk = lane < bs ? yr[c0 + lane] : zero<T>();
            for (int i = bs - 1; i >= 0; --i) {
                const T xi = shfl_div_alpha(yk, i, alpha + c0 + i);
                if (lane == i) yk = xi;
                if (lane < i) yk -= mul(Ablk[(int64_t)i * lda + c0 + lane], xi);
            }
            sx[lane] = yk;
        }
        __syncthreads();
        if (blockIdx.x == 0 && tid < bs) x[(int64_t)rhs * ldx + c0 + tid] = sx[tid];
        for (int64_t r = (int64_t)blockIdx.x * blockDim.x + tid; r < c0; r += (int64_t)gridDim.x * blockDim.x) {
            T acc = zero<T>();
            for (int k = 0; k < bs; ++k) acc += mul(Ablk[(int64_t)k * lda + r], sx[k]);
            yr[r] -= acc;
        }
        __syncthreads();
    }
}

// Forward substitution with R^H (the adjoint solve z = R^{-H} y), column oriented: the mirror of k_backsolve_step.  Every CTA
// solves the bs x bs diagonal block z_i = (y_i - sum_{j<i} conj(R[j,i]) z_j) / conj(alpha_i) (one warp, first row to last), then
// y[r] -= sum_k conj(R[c0 + k, r]) z_k for the rows r in [c0 + bs, n) of its warps (one warp per row: row r of R^H is column r of
// A, so the bs entries it needs are contiguous and a warp reads them in one coalesced load).  CTA 0 publishes z_blk.
// The double2 kernel keeps its minimum of one CTA per SM (0 leaves the double one without a minimum).
template <typename T>
__global__ void __launch_bounds__(256, std::is_same<T, double2>::value ? 1 : 0)
    k_forwardsolve_step(const T* __restrict__ A, int64_t lda, const T* __restrict__ alpha, T* __restrict__ y, int64_t ldy, int nrhs,
                        T* __restrict__ x, int64_t ldx, int64_t c0, int bs, int64_t n) {
    __shared__ T sx[BS_BLK], sD[BS_BLK][BS_BLK + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int e = tid; e < BS_BLK * BS_BLK; e += 256) {                      // sD[j][i] = R[c0 + i, c0 + j], i < j: column j of A
        const int i = e & 31, j = e >> 5;
        sD[j][i] = (i < j && j < bs) ? A[(c0 + j) * lda + c0 + i] : zero<T>();
    }
    __syncthreads();
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        T* yr = y + (int64_t)rhs * ldy;
        if (tid < 32) {
            T yk = lane < bs ? yr[c0 + lane] : zero<T>();
            for (int i = 0; i < bs; ++i) {
                const T zi = div_conj(shfl(yk, i), alpha[c0 + i]);
                if (lane == i) yk = zi;
                if (lane > i) yk -= conj_mul(sD[lane][i], zi);
            }
            sx[lane] = yk;
        }
        __syncthreads();
        if (blockIdx.x == 0 && tid < bs) x[(int64_t)rhs * ldx + c0 + tid] = sx[tid];
        const T zl = lane < bs ? sx[lane] : zero<T>();
        for (int64_t r = c0 + bs + (int64_t)blockIdx.x * 8 + warp; r < n; r += (int64_t)gridDim.x * 8) {
            const T t = lane < bs ? conj_mul(A[r * lda + c0 + lane], zl) : zero<T>();
            const T acc = warp_sum(t);
            if (lane == 0) yr[r] -= acc;
        }
        __syncthreads();
    }
}

// partialdot(a, b, is, ::Type{<:Complex}) (S:51-59): sum conj(a[i]) b[i] over [i0, i1); one CTA.
__global__ void __launch_bounds__(1024, 1) k_partialdot_c(const double2* __restrict__ x, const double2* __restrict__ y, int64_t i0,
                                                          int64_t i1, double2* __restrict__ out) {
    __shared__ double2 red[32];
    const int tid = threadIdx.x;
    double2 acc = make_double2(0.0, 0.0);
    for (int64_t i = i0 + tid; i < i1; i += 1024) {
        const double2 t = cmulc(x[i], y[i]);
        acc.x += t.x;
        acc.y += t.y;
    }
    acc = block_sum2(acc, red, tid, 1024);
    if (tid == 0) *out = acc;
}

}  // namespace dhqr
