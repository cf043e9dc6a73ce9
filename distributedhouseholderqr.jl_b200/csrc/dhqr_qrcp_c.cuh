// dhqr_qrcp_c.cuh — ComplexF64 QR with column pivoting (LAPACK zgeqp3 / zlaqps): A P = Q R in the library's complex storage format
// (H_j = I - v_j v_j^H, ||v_j||^2 = 2, complex alpha; dhqr_complex.cuh).
//
// The scheme of dhqr_qrcp.cuh in complex arithmetic: panels of QP_NB = 32 complex columns, the trailing matrix deferred as
// A - V F^H inside a panel (F: n x 32 complex, F[c, l] = (column c in its deferred state)^H v_l), four launches per column:
//   k_qrcp_pivot_c   argmax of vn1[j:n] (same order, ties and NaN rule as k_qrcp_pivot); columns j and p swapped over all m rows;
//                    x = A[j:, j] - A[j:, k0:j] conj(F[j, 0:jj])' and the partial sums of |x_i|^2; the CTA that arrives last forms
//                    alpha = -exp(i angle(x0)) ||x|| and s = 1 / sqrt(||x|| (||x|| + |x0|)) exactly as k_house1_c does (signed-zero
//                    pivots included), then swaps vn1, vn2, jpvt and the two rows of F
//   k_qrcp_gemv_c    A[j:, k0:n]^H x as per-row-split partials: Re(a^H x) = a_r . x_r and Im(a^H x) = a_r . (-i x)_r, two real
//                    dot products over the same double2 loads; CTAs of column tile 0 write v = s (x - alpha e_0) into A[j:, j]
//   k_qrcp_finish_c  one thread per column c > j: A[j:, c]^H v = s (A[j:, c]^H x - alpha conj(A[j, c])) from the partials,
//                    F[c, jj] = that - F[c, 0:jj] (V[j:, k0:j]^H v), the row update of A[j, c] and the downdate of vn1[c] with |r_jc|
//   k_qrcp_renorm_c  exact norm of each flagged column in its deferred state
// After the panel, A[c1:, c1:] -= V F^H is the real update C += V^ Y^ on the real view (2m x n, leading dimension 2 lda):
// V^ = [v_r, v_i, ...] (k_pack_c) and Y^[2l, c] = -Re F[c, l], Y^[2l+1, c] = +Im F[c, l] (k_qrcp_ypack_c), since the real view of
// v conj(f) is Re f v_r - Im f v_i.
#pragma once
#include "dhqr_complex.cuh"
#include "dhqr_qrcp.cuh"

namespace dhqr {

constexpr int QPC_GCOLS = 16;        // complex columns per CTA of k_qrcp_gemv_c (32 real accumulators, as k_qrcp_gemv)

struct QrcpArgsC {
    double2* A; int64_t lda; int64_t m; int64_t n;
    int64_t j, k0; int jj;           // column in flight, first column of its panel, j - k0
    double2* alpha;                  // diag(R)
    double* vn1; double* vn2;        // partial and reference column norms
    int64_t* jpvt;
    int* flag;                       // columns to renorm
    double2* F; int64_t ldf;         // n x 32
    double2* x;                      // the updated column j, rows j..m-1
    double* part1;                   // k_qrcp_pivot_c: partial sums of |x_i|^2, one per CTA
    double2* part2; int64_t ldp;     // k_qrcp_gemv_c: [split][column - k0]
    int nsplit; int64_t split_rows;  // k_qrcp_gemv_c: row splits
    QrcpCtl* ctl;                    // alpha (real part), alpha_im, scale, ticket, renorm counter
};

__device__ __forceinline__ double2 cmulcb(double2 a, double2 b) {   // a * conj(b)
    return make_double2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
__device__ __forceinline__ double cabs2(double2 a) { return a.x * a.x + a.y * a.y; }

// initial column norms: one CTA per column, jpvt = identity
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_init_c(const double2* __restrict__ A, int64_t lda, int64_t m, double* vn1,
                                                            double* vn2, int64_t* jpvt, int* flag) {
    __shared__ double red[QP_THREADS / 32];
    const int64_t c = blockIdx.x;
    const int tid = threadIdx.x;
    const double2* col = A + c * lda;
    double s = 0.0;
    for (int64_t i = tid; i < m; i += QP_THREADS) s += cabs2(col[i]);
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < QP_THREADS / 32; ++w) t += red[w];
        t = sqrt(t);
        vn1[c] = t; vn2[c] = t; jpvt[c] = c; flag[c] = 0;
    }
}

__global__ void __launch_bounds__(QP_THREADS) k_qrcp_pivot_c(QrcpArgsC a) {
    __shared__ double sv[QP_THREADS / 32];
    __shared__ int64_t si[QP_THREADS / 32];
    __shared__ double2 sF[QP_NB];
    __shared__ double sred[QP_THREADS / 32];
    __shared__ int s_last;
    __shared__ int64_t s_p;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    double bv = -1.0;
    int64_t bi = a.n;
    for (int64_t c = a.j + tid; c < a.n; c += QP_THREADS) {
        const double v = a.vn1[c];
        if (qp_better(v, c, bv, bi)) { bv = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (qp_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
        double v = sv[0];
        int64_t i = si[0];
        for (int w = 1; w < QP_THREADS / 32; ++w)
            if (qp_better(sv[w], si[w], v, i)) { v = sv[w]; i = si[w]; }
        s_p = i;
    }
    __syncthreads();
    const int64_t p = s_p, j = a.j;
    if (tid < a.jj) sF[tid] = a.F[p + tid * a.ldf];
    __syncthreads();
    double2* Aj = a.A + j * a.lda;
    double2* Ap = a.A + p * a.lda;
    const double2* Ak = a.A + a.k0 * a.lda;
    const int64_t r0 = (int64_t)blockIdx.x * QP_PROWS, r1 = min(a.m, r0 + QP_PROWS);
    double ss = 0.0;
    for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
        const double2 aj = Aj[i], ap = Ap[i];
        if (i < j) {
            Aj[i] = ap;
        } else {
            double2 x = ap;
            for (int l = 0; l < a.jj; ++l) {
                const double2 t = cmulcb(Ak[(int64_t)l * a.lda + i], sF[l]);
                x.x -= t.x;
                x.y -= t.y;
            }
            a.x[i - j] = x;
            ss += cabs2(x);
        }
        if (p != j) Ap[i] = aj;
    }
    ss = warp_sum(ss);
    if (lane == 0) sred[warp] = ss;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < QP_THREADS / 32; ++w) t += sred[w];
        a.part1[blockIdx.x] = t;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(&a.ctl->ticket, 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) {
        double t = 0.0;
        for (unsigned g = 0; g < gridDim.x; ++g) t += __ldcg(&a.part1[g]);
        const double vmax = a.vn1[p];
        const double2 x0 = __ldcg(&a.x[0]);
        const double s = sqrt(t);
        double2 al;
        double sc;
        if (vmax == 0.0 || s == 0.0) {           // every remaining column is zero in working precision: H = I
            al = make_double2(0.0, 0.0); sc = 0.0;
        } else {                                 // k_house1_c: alpha = -exp(i angle(x0)) s, angle(+-0 +-0i) = +-0 or +-pi
            const double a0 = hypot(x0.x, x0.y);
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
            al = make_double2(-ux * s, -uy * s);
            sc = 1.0 / sqrt(s * (s + a0));
        }
        a.ctl->alpha = al.x; a.ctl->alpha_im = al.y; a.ctl->scale = sc;
        a.alpha[j] = al;
        if (p != j) {
            double t1 = a.vn1[j]; a.vn1[j] = a.vn1[p]; a.vn1[p] = t1;
            t1 = a.vn2[j]; a.vn2[j] = a.vn2[p]; a.vn2[p] = t1;
            const int64_t t2 = a.jpvt[j]; a.jpvt[j] = a.jpvt[p]; a.jpvt[p] = t2;
        }
        a.ctl->ticket = 0u;
    }
    if (p != j && tid < a.jj) {
        const double2 f = a.F[j + tid * a.ldf];
        a.F[j + tid * a.ldf] = sF[tid];
        a.F[p + tid * a.ldf] = f;
    }
}

// partials of A[j:, k0:n]^H x: grid (column tiles of QPC_GCOLS, row splits); column j contributes nothing (its slot is v)
__global__ void __launch_bounds__(QP_THREADS, 2) k_qrcp_gemv_c(QrcpArgsC a) {
    __shared__ double2 red[QP_THREADS / 32][QPC_GCOLS];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t j = a.j;
    const int64_t c0 = a.k0 + (int64_t)blockIdx.x * QPC_GCOLS;
    const int64_t r0 = j + (int64_t)blockIdx.y * a.split_rows, r1 = min(a.m, r0 + a.split_rows);
    const int ncl = (int)min((int64_t)QPC_GCOLS, a.n - c0);
    const double2* A0 = a.A + c0 * a.lda;
    double re[QPC_GCOLS], im[QPC_GCOLS];
#pragma unroll
    for (int q = 0; q < QPC_GCOLS; ++q) { re[q] = 0.0; im[q] = 0.0; }
    if (ncl == QPC_GCOLS && (j < c0 || j >= c0 + QPC_GCOLS)) {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double2 xi = a.x[i - j];
            double2 v[QPC_GCOLS];
#pragma unroll
            for (int q = 0; q < QPC_GCOLS; ++q) v[q] = A0[(int64_t)q * a.lda + i];
#pragma unroll
            for (int q = 0; q < QPC_GCOLS; ++q) {
                re[q] += v[q].x * xi.x + v[q].y * xi.y;
                im[q] += v[q].x * xi.y - v[q].y * xi.x;
            }
        }
    } else {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double2 xi = a.x[i - j];
#pragma unroll
            for (int q = 0; q < QPC_GCOLS; ++q)
                if (q < ncl && c0 + q != j) {
                    const double2 v = A0[(int64_t)q * a.lda + i];
                    re[q] += v.x * xi.x + v.y * xi.y;
                    im[q] += v.x * xi.y - v.y * xi.x;
                }
        }
    }
#pragma unroll
    for (int q = 0; q < QPC_GCOLS; ++q) {
        const double sr = warp_sum(re[q]), si = warp_sum(im[q]);
        if (lane == q) red[warp][q] = make_double2(sr, si);
    }
    __syncthreads();
    if (tid < ncl) {
        double2 s = make_double2(0.0, 0.0);
        for (int w = 0; w < QP_THREADS / 32; ++w) { s.x += red[w][tid].x; s.y += red[w][tid].y; }
        a.part2[(int64_t)blockIdx.y * a.ldp + (c0 - a.k0) + tid] = s;
    }
    if (blockIdx.x == 0) {
        const double alr = a.ctl->alpha, ali = a.ctl->alpha_im, sc = a.ctl->scale;
        double2* Aj = a.A + j * a.lda;
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            double2 xi = a.x[i - j];
            if (i == j) { xi.x -= alr; xi.y -= ali; }
            Aj[i] = make_double2(xi.x * sc, xi.y * sc);
        }
    }
}

// one thread per column c > j: F column jj, row j of A, downdate of vn1[c]
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_finish_c(QrcpArgsC a) {
    __shared__ double2 g[QP_NB];     // V[j:, k0 + l]^H v, l < jj
    __shared__ double2 vr[QP_NB];    // V[j, k0 + l], l <= jj
    const int tid = threadIdx.x;
    const int64_t j = a.j;
    const double2 al = make_double2(a.ctl->alpha, a.ctl->alpha_im);
    const double sc = a.ctl->scale;
    if (tid < a.jj) {
        double2 s = make_double2(0.0, 0.0);
        for (int q = 0; q < a.nsplit; ++q) { const double2 t = a.part2[(int64_t)q * a.ldp + tid]; s.x += t.x; s.y += t.y; }
        const double2 vj = a.A[j + (a.k0 + tid) * a.lda];
        const double2 t = cmulcb(al, vj);
        g[tid] = make_double2(sc * (s.x - t.x), sc * (s.y - t.y));
        vr[tid] = vj;
    } else if (tid == a.jj) {
        vr[tid] = a.A[j + j * a.lda];
    }
    __syncthreads();
    const int64_t c = j + 1 + (int64_t)blockIdx.x * QP_THREADS + tid;
    if (c >= a.n) return;
    double2 y = make_double2(0.0, 0.0);
    for (int q = 0; q < a.nsplit; ++q) { const double2 t = a.part2[(int64_t)q * a.ldp + (c - a.k0)]; y.x += t.x; y.y += t.y; }
    double2* ajc = a.A + j + c * a.lda;
    const double2 arow = *ajc;
    const double2 t0 = cmulcb(al, arow);
    double2 f = make_double2(sc * (y.x - t0.x), sc * (y.y - t0.y));
    for (int l = 0; l < a.jj; ++l) {
        const double2 t = cmul(a.F[c + l * a.ldf], g[l]);
        f.x -= t.x;
        f.y -= t.y;
    }
    a.F[c + a.jj * a.ldf] = f;
    double2 r = arow;
    for (int l = 0; l < a.jj; ++l) {
        const double2 t = cmulcb(vr[l], a.F[c + l * a.ldf]);
        r.x -= t.x;
        r.y -= t.y;
    }
    const double2 t1 = cmulcb(vr[a.jj], f);
    r.x -= t1.x;
    r.y -= t1.y;
    *ajc = r;
    const double v1 = a.vn1[c];
    if (v1 != 0.0) {                                   // zlaqps: a zero norm is never downdated
        double t = hypot(r.x, r.y) / v1;
        t = fmax(0.0, (1.0 + t) * (1.0 - t));
        const double q = v1 / a.vn2[c];
        if (t * q * q <= 1.4901161193847656e-08) a.flag[c] = 1;   // tol3z = sqrt(eps): renorm exactly
        else a.vn1[c] = v1 * sqrt(t);
    }
}

// exact norm of each flagged column c > j in its deferred state, rows j+1..m-1 (CTAs stride over the columns)
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_renorm_c(QrcpArgsC a) {
    __shared__ double2 sF[QP_NB];
    __shared__ double red[QP_THREADS / 32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nl = a.jj + 1;
    const double2* Ak = a.A + a.k0 * a.lda;
    for (int64_t c = a.j + 1 + blockIdx.x; c < a.n; c += gridDim.x) {
        if (!a.flag[c]) continue;
        __syncthreads();
        if (tid < nl) sF[tid] = a.F[c + tid * a.ldf];
        __syncthreads();
        const double2* col = a.A + c * a.lda;
        double s = 0.0;
        for (int64_t i = a.j + 1 + tid; i < a.m; i += QP_THREADS) {
            double2 v = col[i];
            for (int l = 0; l < nl; ++l) {
                const double2 t = cmulcb(Ak[(int64_t)l * a.lda + i], sF[l]);
                v.x -= t.x;
                v.y -= t.y;
            }
            s += cabs2(v);
        }
        s = warp_sum(s);
        if (lane == 0) red[warp] = s;
        __syncthreads();
        if (tid == 0) {
            double t = 0.0;
            for (int w = 0; w < QP_THREADS / 32; ++w) t += red[w];
            t = sqrt(t);
            a.vn1[c] = t; a.vn2[c] = t; a.flag[c] = 0;
            atomicAdd(&a.ctl->renorms, 1ull);
        }
    }
}

// Y^ of one panel in the ypk layout of the 128-instantiation of C += V Y (nkq_alloc = 4 k-chunks per column tile, the first two
// written: real k index kk = 2l + (0: real part, 1: imaginary part) of reflector l): Y^[2l, c] = -Re F[c0 + c, l],
// Y^[2l + 1, c] = +Im F[c0 + c, l] for l < kb and c < ncols, zero elsewhere (padding included)
constexpr int QPC_NKQ = 2 * QP_NB / KC;                    // k-chunks of Y^ the update runs
__global__ void k_qrcp_ypack_c(const double2* __restrict__ F, int64_t ldf, int64_t c0, int ncols, int kb, double* __restrict__ ypk) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t tiles = (ncols + YT - 1) / YT;
    if (t >= tiles * QPC_NKQ * YT * LDK) return;
    const int k = (int)(t % LDK);
    const int64_t col = (t / LDK) % YT;
    const int kq = (int)((t / ((int64_t)YT * LDK)) % QPC_NKQ);
    const int64_t tile = t / ((int64_t)QPC_NKQ * YT * LDK);
    const int kk = kq * KC + k, l = kk >> 1;
    const int64_t cc = tile * YT + col;
    double v = 0.0;
    if (k < KC && l < kb && cc < ncols) {
        const double2 f = F[c0 + cc + (int64_t)l * ldf];
        v = (kk & 1) ? f.y : -f.x;
    }
    ypk[(tile * (VPK_COLS / KC) + kq) * (YT * LDK) + col * LDK + k] = v;
}

// basic solution: b[jpvt[i]] = z[i] for i < rank, 0 for rank <= i < n; jpvt entries outside [0, n) are skipped
__global__ void k_qrcp_scatter_c(const double2* __restrict__ z, int64_t ldz, const int64_t* __restrict__ jpvt, int64_t n, int64_t rank,
                                 double2* __restrict__ b, int64_t ldb) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t d = jpvt[i];
    if (d < 0 || d >= n) return;
    b[d + (int64_t)blockIdx.y * ldb] = i < rank ? z[i + (int64_t)blockIdx.y * ldz] : make_double2(0.0, 0.0);
}

// dhqr_cod_c64: F (n x rank) <- R_r^H with a conjugating transpose: F[j, i] = conj(A[i, j]) for j > i, conj(alpha[i]) for j = i and 0
// for j < i.  Tiles as k_cod_pack; the reflectors below A's diagonal are never read.
__global__ void __launch_bounds__(CP_TILE * CP_ROWS) k_cod_pack_c(const double2* __restrict__ A, int64_t lda, const double2* __restrict__ alpha,
                                                                  int64_t n, int64_t rank, double2* __restrict__ F, int64_t ldf) {
    __shared__ double2 t[CP_TILE][CP_TILE + 1];                        // t[j - j0][i - i0]
    const int64_t j0 = (int64_t)blockIdx.x * CP_TILE, i0 = (int64_t)blockIdx.y * CP_TILE;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const bool lower = j0 + CP_TILE - 1 >= i0;
    if (lower) {
        for (int r = ty; r < CP_TILE; r += CP_ROWS) {
            const int64_t j = j0 + r, i = i0 + tx;
            double2 v = make_double2(0.0, 0.0);
            if (j < n && i < rank && j >= i) {
                const double2 z = j > i ? A[i + j * lda] : alpha[i];
                v = make_double2(z.x, -z.y);
            }
            t[r][tx] = v;
        }
        __syncthreads();
    }
    for (int r = ty; r < CP_TILE; r += CP_ROWS) {
        const int64_t i = i0 + r, j = j0 + tx;
        if (i < rank && j < n) F[j + i * ldf] = lower ? t[tx][r] : make_double2(0.0, 0.0);
    }
}

}  // namespace dhqr
