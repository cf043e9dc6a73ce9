// dhqr_qrcp.cuh — Householder QR with column pivoting (LAPACK dgeqp3 / dlaqps, Quintana-Orti, Sun and Bischof): A P = Q R.
//
// Panels of QP_NB = 32 columns.  Inside a panel the trailing matrix is left in a deferred state, A - V F' (F: n x 32, one
// column per reflector), and every column step is four launches:
//   k_qrcp_pivot  p = argmax vn1[j:n] (every CTA computes it, in the same fixed order); columns j and p swapped over all m rows;
//                 the new column brought up to date, x = A[j:, j] - A[j:, k0:j] F[j, 0:jj]', into a contiguous buffer, with the
//                 partial sums of squares; the CTA that arrives last forms alpha and the scale of v and swaps vn1, vn2, jpvt and
//                 the two rows of F (which every CTA read before it arrived)
//   k_qrcp_gemv   the F-column GEMV, A[j:, k0:n]' x over the stored trailing matrix (column j skipped), as per-row-split
//                 partials; CTAs of column tile 0 write v = s (x - alpha e_0) into A[j:, j]
//   k_qrcp_finish one thread per column c > j: A[j:, c]' v = s (A[j:, c]' x - alpha A[j, c]) from the partials,
//                 F[c, jj] = that - F[c, 0:jj] (V[j:, k0:j]' v), the row update of A[j, c] and the downdate of vn1[c]
//                 (LAPACK dlaqps); a column whose downdate fails the tol3z test is flagged
//   k_qrcp_renorm every flagged column gets its exact norm in the deferred state, ||A[j+1:, c] - V[j+1:, k0:j+1] F[c, 0:jj+1]'||
// After the panel, A[k0+32:, k0+32:] -= V F' goes through the 32-wide C += V Y kernel with Y = -F' (k_qrcp_ypack).
// No value ever travels to the host: the pivot and every scalar stay on the device, so the driver is one static loop.
// Every reduction runs in a fixed order: two runs give bitwise identical results.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace dhqr {

constexpr int QP_NB = 32;            // panel width (columns of F)
constexpr int QP_THREADS = 256;
constexpr int QP_PROWS = 512;        // rows per CTA of k_qrcp_pivot
constexpr int QP_GCOLS = 32;         // columns per CTA of k_qrcp_gemv

struct QrcpCtl {
    double alpha, scale;             // of the reflector in flight
    unsigned int ticket;             // k_qrcp_pivot: zero on entry, zero again on exit
    unsigned int pad;
    unsigned long long renorms;      // exact renorms since the handle was created
};

struct QrcpArgs {
    double* A; int64_t lda; int64_t m; int64_t n;
    int64_t j, k0; int jj;           // column in flight, first column of its panel, j - k0
    double* alpha;                   // diag(R)
    double* vn1; double* vn2;        // partial and reference column norms
    int64_t* jpvt;
    int* flag;                       // columns to renorm
    double* F; int64_t ldf;          // n x 32
    double* x;                       // the updated column j, rows j..m-1
    double* part1;                   // k_qrcp_pivot: partial sums of squares, one per CTA
    double* part2; int64_t ldp;      // k_qrcp_gemv: [split][column - k0]
    int nsplit; int64_t split_rows;  // k_qrcp_gemv: row splits
    QrcpCtl* ctl;
};

// b beats a: NaN beats every number (numpy argmax), a larger value beats a smaller one, a tie goes to the smaller index (idamax)
__device__ __forceinline__ bool qp_better(double bv, int64_t bi, double av, int64_t ai) {
    if (isnan(bv)) return !isnan(av) || bi < ai;
    if (isnan(av)) return false;
    return bv > av || (bv == av && bi < ai);
}

// initial column norms: one CTA per column, jpvt = identity
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_init(const double* __restrict__ A, int64_t lda, int64_t m, double* vn1,
                                                          double* vn2, int64_t* jpvt, int* flag) {
    __shared__ double red[QP_THREADS / 32];
    const int64_t c = blockIdx.x;
    const int tid = threadIdx.x;
    const double* col = A + c * lda;
    double s = 0.0;
    for (int64_t i = tid; i < m; i += QP_THREADS) { const double v = col[i]; s += v * v; }
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

__global__ void __launch_bounds__(QP_THREADS) k_qrcp_pivot(QrcpArgs a) {
    __shared__ double sv[QP_THREADS / 32];
    __shared__ int64_t si[QP_THREADS / 32];
    __shared__ double sF[QP_NB];
    __shared__ double sred[QP_THREADS / 32];
    __shared__ int s_last;
    __shared__ int64_t s_p;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // argmax over vn1[j:n], scanned in index order per thread, then a fixed tree
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
    // swap columns j and p over this CTA's rows; rows >= j of the pivot column get the panel's column update
    double* Aj = a.A + j * a.lda;
    double* Ap = a.A + p * a.lda;
    const double* Ak = a.A + a.k0 * a.lda;
    const int64_t r0 = (int64_t)blockIdx.x * QP_PROWS, r1 = min(a.m, r0 + QP_PROWS);
    double ss = 0.0;
    for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
        const double aj = Aj[i], ap = Ap[i];
        if (i < j) {
            Aj[i] = ap;
        } else {
            double x = ap;
            for (int l = 0; l < a.jj; ++l) x -= Ak[(int64_t)l * a.lda + i] * sF[l];
            a.x[i - j] = x;
            ss += x * x;
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
    // the CTA that arrived last: every CTA has read vn1 and row p of F, so they can move now
    if (tid == 0) {
        double t = 0.0;
        for (unsigned g = 0; g < gridDim.x; ++g) t += __ldcg(&a.part1[g]);
        const double vmax = a.vn1[p];
        const double x0 = __ldcg(&a.x[0]);
        const double nrm = sqrt(t);
        double al, sc;
        if (vmax == 0.0 || nrm == 0.0) {         // every remaining column is zero in working precision: H = I
            al = 0.0; sc = 0.0;
        } else {
            al = x0 >= 0.0 ? -nrm : nrm;           // a zero leading entry counts as positive
            sc = 1.0 / sqrt(nrm * (nrm + fabs(x0)));
        }
        a.ctl->alpha = al; a.ctl->scale = sc;
        a.alpha[j] = al;
        if (p != j) {
            double t1 = a.vn1[j]; a.vn1[j] = a.vn1[p]; a.vn1[p] = t1;
            t1 = a.vn2[j]; a.vn2[j] = a.vn2[p]; a.vn2[p] = t1;
            const int64_t t2 = a.jpvt[j]; a.jpvt[j] = a.jpvt[p]; a.jpvt[p] = t2;
        }
        a.ctl->ticket = 0u;
    }
    if (p != j && tid < a.jj) {
        const double f = a.F[j + tid * a.ldf];
        a.F[j + tid * a.ldf] = sF[tid];
        a.F[p + tid * a.ldf] = f;
    }
}

// partials of A[j:, k0:n]' x: grid (column tiles of QP_GCOLS, row splits); column j contributes nothing (its slot is v)
__global__ void __launch_bounds__(QP_THREADS, 2) k_qrcp_gemv(QrcpArgs a) {
    __shared__ double red[QP_THREADS / 32][QP_GCOLS];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t j = a.j;
    const int64_t c0 = a.k0 + (int64_t)blockIdx.x * QP_GCOLS;
    const int64_t r0 = j + (int64_t)blockIdx.y * a.split_rows, r1 = min(a.m, r0 + a.split_rows);
    const int ncl = (int)min((int64_t)QP_GCOLS, a.n - c0);
    const double* A0 = a.A + c0 * a.lda;
    double acc[QP_GCOLS];
#pragma unroll
    for (int q = 0; q < QP_GCOLS; ++q) acc[q] = 0.0;
    if (ncl == QP_GCOLS && (j < c0 || j >= c0 + QP_GCOLS)) {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double xi = a.x[i - j];
            double v[QP_GCOLS];
#pragma unroll
            for (int q = 0; q < QP_GCOLS; ++q) v[q] = A0[(int64_t)q * a.lda + i];
#pragma unroll
            for (int q = 0; q < QP_GCOLS; ++q) acc[q] += v[q] * xi;
        }
    } else {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double xi = a.x[i - j];
#pragma unroll
            for (int q = 0; q < QP_GCOLS; ++q)
                if (q < ncl && c0 + q != j) acc[q] += A0[(int64_t)q * a.lda + i] * xi;
        }
    }
#pragma unroll
    for (int q = 0; q < QP_GCOLS; ++q) {
        const double s = warp_sum(acc[q]);
        if (lane == q) red[warp][q] = s;
    }
    __syncthreads();
    if (tid < ncl) {
        double s = 0.0;
        for (int w = 0; w < QP_THREADS / 32; ++w) s += red[w][tid];
        a.part2[(int64_t)blockIdx.y * a.ldp + (c0 - a.k0) + tid] = s;
    }
    if (blockIdx.x == 0) {
        const double al = a.ctl->alpha, sc = a.ctl->scale;
        double* Aj = a.A + j * a.lda;
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double xi = a.x[i - j];
            Aj[i] = (i == j ? xi - al : xi) * sc;
        }
    }
}

// one thread per column c > j: F column jj, row j of A, downdate of vn1[c]
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_finish(QrcpArgs a) {
    __shared__ double g[QP_NB];      // V[j:, k0 + l]' v, l < jj
    __shared__ double vr[QP_NB];     // V[j, k0 + l], l <= jj
    const int tid = threadIdx.x;
    const int64_t j = a.j;
    const double al = a.ctl->alpha, sc = a.ctl->scale;
    if (tid < a.jj) {
        double s = 0.0;
        for (int q = 0; q < a.nsplit; ++q) s += a.part2[(int64_t)q * a.ldp + tid];
        const double vj = a.A[j + (a.k0 + tid) * a.lda];
        g[tid] = sc * (s - al * vj);
        vr[tid] = vj;
    } else if (tid == a.jj) {
        vr[tid] = a.A[j + j * a.lda];
    }
    __syncthreads();
    const int64_t c = j + 1 + (int64_t)blockIdx.x * QP_THREADS + tid;
    if (c >= a.n) return;
    double y = 0.0;
    for (int q = 0; q < a.nsplit; ++q) y += a.part2[(int64_t)q * a.ldp + (c - a.k0)];
    double* ajc = a.A + j + c * a.lda;
    const double arow = *ajc;
    double f = sc * (y - al * arow);
    for (int l = 0; l < a.jj; ++l) f -= a.F[c + l * a.ldf] * g[l];
    a.F[c + a.jj * a.ldf] = f;
    double r = arow;
    for (int l = 0; l < a.jj; ++l) r -= vr[l] * a.F[c + l * a.ldf];
    r -= vr[a.jj] * f;
    *ajc = r;
    const double v1 = a.vn1[c];
    if (v1 != 0.0) {                                   // dlaqps: a zero norm is never downdated
        double t = fabs(r) / v1;
        t = fmax(0.0, (1.0 + t) * (1.0 - t));
        const double q = v1 / a.vn2[c];
        if (t * q * q <= 1.4901161193847656e-08) a.flag[c] = 1;   // tol3z = sqrt(eps): renorm exactly
        else a.vn1[c] = v1 * sqrt(t);
    }
}

// exact norm of each flagged column c > j in its deferred state, rows j+1..m-1 (CTAs stride over the columns)
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_renorm(QrcpArgs a) {
    __shared__ double sF[QP_NB];
    __shared__ double red[QP_THREADS / 32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nl = a.jj + 1;
    const double* Ak = a.A + a.k0 * a.lda;
    for (int64_t c = a.j + 1 + blockIdx.x; c < a.n; c += gridDim.x) {
        if (!a.flag[c]) continue;
        __syncthreads();
        if (tid < nl) sF[tid] = a.F[c + tid * a.ldf];
        __syncthreads();
        const double* col = a.A + c * a.lda;
        double s = 0.0;
        for (int64_t i = a.j + 1 + tid; i < a.m; i += QP_THREADS) {
            double v = col[i];
            for (int l = 0; l < nl; ++l) v -= Ak[(int64_t)l * a.lda + i] * sF[l];
            s += v * v;
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

// Y = -F' of one panel in the ypk layout of the 32-wide C += V Y kernel (nkq_alloc = 1): rows c >= c0 of F, columns l < kb
__global__ void k_qrcp_ypack(const double* __restrict__ F, int64_t ldf, int64_t c0, int ncols, int kb, double* __restrict__ ypk) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t tot = (int64_t)((ncols + YT - 1) / YT) * YT * LDK;
    if (t >= tot) return;
    const int l = (int)(t % LDK);
    const int64_t col = (t / LDK) % YT + (t / ((int64_t)YT * LDK)) * YT;
    ypk[t] = (l < kb && col < ncols) ? -F[c0 + col + (int64_t)l * ldf] : 0.0;
}

// basic solution: b[jpvt[i]] = z[i] for i < rank, 0 for rank <= i < n; jpvt entries outside [0, n) are skipped
__global__ void k_qrcp_scatter(const double* __restrict__ z, int64_t ldz, const int64_t* __restrict__ jpvt, int64_t n, int64_t rank,
                               double* __restrict__ b, int64_t ldb) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t d = jpvt[i];
    if (d < 0 || d >= n) return;
    b[d + (int64_t)blockIdx.y * ldb] = i < rank ? z[i + (int64_t)blockIdx.y * ldz] : 0.0;
}

}  // namespace dhqr
