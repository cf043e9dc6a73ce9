// dhqr_complex.cuh — ComplexF64 path (the reference tests both element types, test/runtests.jl:43; S:9, S:51-59, S:162-196).
//
// A complex reflector H = I - v v^H with |v|^2 = 2 acts on the REAL view of a complex column (re, im interleaved, length 2m) as
// the product of two commuting real reflectors: with v_r = [x0, y0, x1, y1, ...] and v_i = i v = [-y0, x0, -y1, x1, ...]
//     Re(v^H c) = v_r . c_r,   Im(v^H c) = v_i . c_r,   c - v s = c_r - (Re s) v_r - (Im s) v_i,   v_r . v_i = 0, |v_r|^2 = |v_i|^2 = 2
// (partialdot S:51-59 and hotloop! S:162-196 written out in reals).  So the trailing update of a panel of kb complex
// reflectors IS the real block-reflector update with V^ = [v1_r, v1_i, v2_r, v2_i, ...] (2 kb real vectors) on the real view of
// the trailing matrix (2m x n, leading dimension 2 lda), T^{-1} = I + striu(V^' V^): the fp64 tensor-pipe GEMM pair of the real
// path is reused as is (this is the 4M real decomposition of the complex rank-k update).  New here: the complex panel
// factorisation (column by column, S:127-135 with alphafactor(::Complex) S:9), the packing of V^, the complex back-substitution
// (S:256-282) and the conjugating partialdot primitive.
#pragma once
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

// S:129-135 for one complex column (one CTA): s = |x|, alpha = -exp(i angle(x0)) s  (S:9), f = 1 / sqrt(s (s + |x0|)),
// x0 -= alpha, x *= f.  angle = atan2(im, re) sees the signs of a zero pivot: angle(+0 +- 0i) = +-0 gives alpha = -s,
// angle(-0 +- 0i) = +-pi gives alpha = -s (cos pi, +-sin pi) = s (1, -+1.2246e-16).
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
        const double a0 = hypot(x0.x, x0.y);
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
        const double2 al = make_double2(-ux * s, -uy * s);
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

// back-substitution step (S:256-282) for complex R = triu(A,1) + diag(alpha): like k_backsolve_step
__global__ void __launch_bounds__(256) k_backsolve_step_c(const double2* __restrict__ Ablk, int64_t lda, const double2* __restrict__ alpha,
                                                          double2* __restrict__ y, int64_t ldy, int nrhs, double2* __restrict__ x,
                                                          int64_t ldx, int64_t c0, int bs) {
    __shared__ double2 sx[BS_BLK];
    const int tid = threadIdx.x, lane = tid & 31;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        double2* yr = y + (int64_t)rhs * ldy;
        if (tid < 32) {
            double2 yk = lane < bs ? yr[c0 + lane] : make_double2(0.0, 0.0);
            for (int i = bs - 1; i >= 0; --i) {
                const double2 al = alpha[c0 + i];
                const double den = al.x * al.x + al.y * al.y;
                const double nx = __shfl_sync(0xffffffffu, yk.x, i), ny = __shfl_sync(0xffffffffu, yk.y, i);
                const double2 xi = make_double2((nx * al.x + ny * al.y) / den, (ny * al.x - nx * al.y) / den);   // (nx + i ny) / alpha
                if (lane == i) yk = xi;
                if (lane < i) {
                    const double2 t = cmul(Ablk[(int64_t)i * lda + c0 + lane], xi);
                    yk.x -= t.x;
                    yk.y -= t.y;
                }
            }
            sx[lane] = yk;
        }
        __syncthreads();
        if (blockIdx.x == 0 && tid < bs) x[(int64_t)rhs * ldx + c0 + tid] = sx[tid];
        for (int64_t r = (int64_t)blockIdx.x * blockDim.x + tid; r < c0; r += (int64_t)gridDim.x * blockDim.x) {
            double2 acc = make_double2(0.0, 0.0);
            for (int k = 0; k < bs; ++k) {
                const double2 t = cmul(Ablk[(int64_t)k * lda + r], sx[k]);
                acc.x += t.x;
                acc.y += t.y;
            }
            yr[r].x -= acc.x;
            yr[r].y -= acc.y;
        }
        __syncthreads();
    }
}

// n / conj(a) by Smith's algorithm: the ratio of the smaller to the larger part of a is formed first, so neither |a|^2 nor a
// partial product overflows or underflows when n and a lie many decades apart (columns scaled by 10^+-120).  a = 0 gives NaN.
__device__ __forceinline__ double2 cdiv_conj(double2 n, double2 a) {
    const double p = a.x, q = -a.y;                                          // conj(a) = p + i q
    if (fabs(p) >= fabs(q)) {
        const double r = q / p, d = p + q * r;
        return make_double2((n.x + n.y * r) / d, (n.y - n.x * r) / d);
    }
    const double r = p / q, d = q + p * r;
    return make_double2((n.x * r + n.y) / d, (n.y * r - n.x) / d);
}

// forward substitution with R^H (z = R^{-H} y) for complex R = triu(A,1) + diag(alpha): like k_forwardsolve_step, with the
// conjugated products z_i = (y_i - sum_{j<i} conj(R[j,i]) z_j) / conj(alpha_i)
__global__ void __launch_bounds__(256, 1) k_forwardsolve_step_c(const double2* __restrict__ A, int64_t lda, const double2* __restrict__ alpha,
                                                             double2* __restrict__ y, int64_t ldy, int nrhs, double2* __restrict__ x,
                                                             int64_t ldx, int64_t c0, int bs, int64_t n) {
    __shared__ double2 sx[BS_BLK], sD[BS_BLK][BS_BLK + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int e = tid; e < BS_BLK * BS_BLK; e += 256) {                      // sD[j][i] = R[c0 + i, c0 + j], i < j: column j of A
        const int i = e & 31, j = e >> 5;
        sD[j][i] = (i < j && j < bs) ? A[(c0 + j) * lda + c0 + i] : make_double2(0.0, 0.0);
    }
    __syncthreads();
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        double2* yr = y + (int64_t)rhs * ldy;
        if (tid < 32) {
            double2 yk = lane < bs ? yr[c0 + lane] : make_double2(0.0, 0.0);
            for (int i = 0; i < bs; ++i) {
                const double nx = __shfl_sync(0xffffffffu, yk.x, i), ny = __shfl_sync(0xffffffffu, yk.y, i);
                const double2 zi = cdiv_conj(make_double2(nx, ny), alpha[c0 + i]);
                if (lane == i) yk = zi;
                if (lane > i) {
                    const double2 t = cmulc(sD[lane][i], zi);
                    yk.x -= t.x;
                    yk.y -= t.y;
                }
            }
            sx[lane] = yk;
        }
        __syncthreads();
        if (blockIdx.x == 0 && tid < bs) x[(int64_t)rhs * ldx + c0 + tid] = sx[tid];
        const double2 zl = lane < bs ? sx[lane] : make_double2(0.0, 0.0);
        for (int64_t r = c0 + bs + (int64_t)blockIdx.x * 8 + warp; r < n; r += (int64_t)gridDim.x * 8) {
            const double2 t = lane < bs ? cmulc(A[r * lda + c0 + lane], zl) : make_double2(0.0, 0.0);
            const double sre = warp_sum(t.x), sim = warp_sum(t.y);
            if (lane == 0) {
                yr[r].x -= sre;
                yr[r].y -= sim;
            }
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
