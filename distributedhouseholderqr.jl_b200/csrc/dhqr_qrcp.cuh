// dhqr_qrcp.cuh — Householder QR with column pivoting (LAPACK ?geqp3 / ?laqps, Quintana-Orti, Sun and Bischof): A P = Q R, for
// Float64 (T = double) and ComplexF64 (T = double2, in the library's complex storage format: H_j = I - v_j v_j^H, ||v_j||^2 = 2,
// complex alpha; dhqr_complex.cuh).  For double, ^H is ' and conj is the identity.
//
// Panels of QP_NB = 32 columns.  Inside a panel the trailing matrix is left in a deferred state, A - V F^H (F: n x 32, one
// column per reflector, F[c, l] = (column c in its deferred state)^H v_l), and every column step is four launches:
//   k_qrcp_pivot  p = argmax vn1[j:n] (every CTA computes it, in the same fixed order); columns j and p swapped over all m rows;
//                 the new column brought up to date, x = A[j:, j] - A[j:, k0:j] conj(F[j, 0:jj])', into a contiguous buffer,
//                 with the partial sums of |x_i|^2; the CTA that arrives last forms alpha and the scale of v (qp_alpha) and
//                 swaps vn1, vn2, jpvt and the two rows of F (which every CTA read before it arrived)
//   k_qrcp_gemv   the F-column GEMV, A[j:, k0:n]^H x over the stored trailing matrix (column j skipped), as per-row-split
//                 partials; CTAs of column tile 0 write v = s (x - alpha e_0) into A[j:, j]
//   k_qrcp_finish one thread per column c > j: A[j:, c]^H v = s (A[j:, c]^H x - alpha conj(A[j, c])) from the partials,
//                 F[c, jj] = that - F[c, 0:jj] (V[j:, k0:j]^H v), the row update of A[j, c] and the downdate of vn1[c] with
//                 |r_jc| (LAPACK ?laqps); a column whose downdate fails the tol3z test is flagged
//   k_qrcp_renorm every flagged column gets its exact norm in the deferred state, ||A[j+1:, c] - V[j+1:, k0:j+1] F[c, 0:jj+1]^H||
// No value ever travels to the host: the pivot and every scalar stay on the device, so the driver is one static loop.
// Every reduction runs in a fixed order: two runs give bitwise identical results.
//
// k_qrcp_init, k_qrcp_pivot, k_qrcp_renorm, k_qrcp_scatter and k_cod_pack are written once for both types; what differs between
// them is in the overloaded helpers below:
//   alpha         double: -sign(x0) ||x||, a zero x0 counting as positive; double2: -exp(i angle(x0)) ||x|| with k_house1_c's
//                 signed-zero rules (house_alpha), so (A, alpha) is valid input to every other _c64 entry point
//   products      a conj(b), |x|^2; conj is the identity for double
// k_qrcp_gemv and k_qrcp_finish are one overload per type.  The double2 ones are the double ones written out in components (two
// real dot products over the same double2 loads in the GEMV, 16 complex columns per CTA: 32 real accumulators either way, and
// hypot for |r_jc|); every shared formulation tried compiled to the same arithmetic with a different register assignment.
// After each panel, A[k0+32:, k0+32:] -= V F^H.  double: the 32-wide C += V Y kernel with Y = -F' (k_qrcp_ypack).  double2: the
// real C += V^ Y^ on the real view (2m x n, leading dimension 2 lda) through the 128-instantiation, V^ = [v_r, v_i, ...]
// (k_pack_c) and Y^[2l, c] = -Re F[c, l], Y^[2l+1, c] = +Im F[c, l] (k_qrcp_ypack_c), since the real view of v conj(f) is
// Re f v_r - Im f v_i.
// Every double2 expression is the double one in components, in the same order of operations, so the generated code of each type
// is what it was when the two were written separately.
#pragma once
#include "dhqr_complex.cuh"

namespace dhqr {

constexpr int QP_NB = 32;            // panel width (columns of F)
constexpr int QP_THREADS = 256;
constexpr int QP_PROWS = 512;        // rows per CTA of k_qrcp_pivot
template <typename T>
constexpr int QP_GCOLS = 32 * (int)sizeof(double) / (int)sizeof(T);   // columns per CTA of k_qrcp_gemv: 32 real accumulators

struct QrcpCtl {
    double alpha, scale;             // of the reflector in flight
    unsigned int ticket;             // k_qrcp_pivot: zero on entry, zero again on exit
    unsigned int pad;
    unsigned long long renorms;      // exact renorms since the handle was created
    double alpha_im;                 // T = double2: imaginary part of the alpha in flight
};

template <typename T>
struct QrcpArgs {
    T* A; int64_t lda; int64_t m; int64_t n;
    int64_t j, k0; int jj;           // column in flight, first column of its panel, j - k0
    T* alpha;                        // diag(R)
    double* vn1; double* vn2;        // partial and reference column norms
    int64_t* jpvt;
    int* flag;                       // columns to renorm
    T* F; int64_t ldf;               // n x 32
    T* x;                            // the updated column j, rows j..m-1
    double* part1;                   // k_qrcp_pivot: partial sums of |x_i|^2, one per CTA
    T* part2; int64_t ldp;           // k_qrcp_gemv: [split][column - k0]
    int nsplit; int64_t split_rows;  // k_qrcp_gemv: row splits
    QrcpCtl* ctl;
};

__device__ __forceinline__ double qp_abs2(double v) { return v * v; }
__device__ __forceinline__ double qp_abs2(double2 v) { return v.x * v.x + v.y * v.y; }

__device__ __forceinline__ double2 cmulcb(double2 a, double2 b) {   // a * conj(b)
    return make_double2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
// a conj(b)
__device__ __forceinline__ double qp_mul_conj(double a, double b) { return a * b; }
__device__ __forceinline__ double2 qp_mul_conj(double2 a, double2 b) { return cmulcb(a, b); }

// alpha and the scale 1 / sqrt(nrm (nrm + |x0|)) of the reflector of a column with leading entry x0 and norm nrm > 0; for double2
// alpha is k_house1_c's (house_alpha, dhqr_complex.cuh)
__device__ __forceinline__ void qp_alpha(double x0, double nrm, double& alpha, double& scale) {
    alpha = x0 >= 0.0 ? -nrm : nrm;           // a zero leading entry counts as positive
    scale = 1.0 / sqrt(nrm * (nrm + fabs(x0)));
}
__device__ __forceinline__ void qp_alpha(double2 x0, double nrm, double2& alpha, double& scale) {
    double a0;
    alpha = house_alpha(x0, nrm, a0);
    scale = 1.0 / sqrt(nrm * (nrm + a0));
}

// the alpha in flight, in QrcpCtl
__device__ __forceinline__ void qp_put_alpha(QrcpCtl* c, double al) { c->alpha = al; }
__device__ __forceinline__ void qp_put_alpha(QrcpCtl* c, double2 al) { c->alpha = al.x; c->alpha_im = al.y; }

// k_cod_pack: entry (j, i) of R_r^H, zero outside it (i >= rank or j >= n)
__device__ __forceinline__ double qp_rrh(const double* A, int64_t lda, const double* alpha, int64_t n, int64_t rank, int64_t i,
                                         int64_t j) {
    double v = 0.0;
    if (j < n && i < rank) v = j > i ? A[i + j * lda] : (j == i ? alpha[i] : 0.0);
    return v;
}
__device__ __forceinline__ double2 qp_rrh(const double2* A, int64_t lda, const double2* alpha, int64_t n, int64_t rank, int64_t i,
                                          int64_t j) {
    double2 v = make_double2(0.0, 0.0);
    if (j < n && i < rank && j >= i) {
        const double2 z = j > i ? A[i + j * lda] : alpha[i];
        v = make_double2(z.x, -z.y);
    }
    return v;
}

// b beats a: NaN beats every number (numpy argmax), a larger value beats a smaller one, a tie goes to the smaller index (idamax)
__device__ __forceinline__ bool qp_better(double bv, int64_t bi, double av, int64_t ai) {
    if (isnan(bv)) return !isnan(av) || bi < ai;
    if (isnan(av)) return false;
    return bv > av || (bv == av && bi < ai);
}

// initial column norms: one CTA per column, jpvt = identity
template <typename T>
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_init(const T* __restrict__ A, int64_t lda, int64_t m, double* vn1, double* vn2,
                                                          int64_t* jpvt, int* flag) {
    __shared__ double red[QP_THREADS / 32];
    const int64_t c = blockIdx.x;
    const int tid = threadIdx.x;
    const T* col = A + c * lda;
    double s = 0.0;
    for (int64_t i = tid; i < m; i += QP_THREADS) s += qp_abs2(col[i]);
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

template <typename T>
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_pivot(QrcpArgs<T> a) {
    __shared__ double sv[QP_THREADS / 32];
    __shared__ int64_t si[QP_THREADS / 32];
    __shared__ T sF[QP_NB];
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
    T* Aj = a.A + j * a.lda;
    T* Ap = a.A + p * a.lda;
    const T* Ak = a.A + a.k0 * a.lda;
    const int64_t r0 = (int64_t)blockIdx.x * QP_PROWS, r1 = min(a.m, r0 + QP_PROWS);
    double ss = 0.0;
    for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
        const T aj = Aj[i], ap = Ap[i];
        if (i < j) {
            Aj[i] = ap;
        } else {
            T x = ap;
            for (int l = 0; l < a.jj; ++l) x -= qp_mul_conj(Ak[(int64_t)l * a.lda + i], sF[l]);
            a.x[i - j] = x;
            ss += qp_abs2(x);
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
        const T x0 = __ldcg(&a.x[0]);
        const double nrm = sqrt(t);
        T al;
        double sc;
        if (vmax == 0.0 || nrm == 0.0) {         // every remaining column is zero in working precision: H = I
            al = zero<T>(); sc = 0.0;
        } else {
            qp_alpha(x0, nrm, al, sc);
        }
        qp_put_alpha(a.ctl, al); a.ctl->scale = sc;
        a.alpha[j] = al;
        if (p != j) {
            double t1 = a.vn1[j]; a.vn1[j] = a.vn1[p]; a.vn1[p] = t1;
            t1 = a.vn2[j]; a.vn2[j] = a.vn2[p]; a.vn2[p] = t1;
            const int64_t t2 = a.jpvt[j]; a.jpvt[j] = a.jpvt[p]; a.jpvt[p] = t2;
        }
        a.ctl->ticket = 0u;
    }
    if (p != j && tid < a.jj) {
        const T f = a.F[j + tid * a.ldf];
        a.F[j + tid * a.ldf] = sF[tid];
        a.F[p + tid * a.ldf] = f;
    }
}

// partials of A[j:, k0:n]' x: grid (column tiles of QP_GCOLS<double>, row splits); column j contributes nothing (its slot is v)
__global__ void __launch_bounds__(QP_THREADS, 2) k_qrcp_gemv(QrcpArgs<double> a) {
    __shared__ double red[QP_THREADS / 32][QP_GCOLS<double>];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t j = a.j;
    const int64_t c0 = a.k0 + (int64_t)blockIdx.x * QP_GCOLS<double>;
    const int64_t r0 = j + (int64_t)blockIdx.y * a.split_rows, r1 = min(a.m, r0 + a.split_rows);
    const int ncl = (int)min((int64_t)QP_GCOLS<double>, a.n - c0);
    const double* A0 = a.A + c0 * a.lda;
    double acc[QP_GCOLS<double>];
#pragma unroll
    for (int q = 0; q < QP_GCOLS<double>; ++q) acc[q] = 0.0;
    if (ncl == QP_GCOLS<double> && (j < c0 || j >= c0 + QP_GCOLS<double>)) {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double xi = a.x[i - j];
            double v[QP_GCOLS<double>];
#pragma unroll
            for (int q = 0; q < QP_GCOLS<double>; ++q) v[q] = A0[(int64_t)q * a.lda + i];
#pragma unroll
            for (int q = 0; q < QP_GCOLS<double>; ++q) acc[q] += v[q] * xi;
        }
    } else {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double xi = a.x[i - j];
#pragma unroll
            for (int q = 0; q < QP_GCOLS<double>; ++q)
                if (q < ncl && c0 + q != j) acc[q] += A0[(int64_t)q * a.lda + i] * xi;
        }
    }
#pragma unroll
    for (int q = 0; q < QP_GCOLS<double>; ++q) {
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
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_finish(QrcpArgs<double> a) {
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

// partials of A[j:, k0:n]^H x: grid (column tiles of QP_GCOLS<double2>, row splits); column j contributes nothing (its slot is v)
__global__ void __launch_bounds__(QP_THREADS, 2) k_qrcp_gemv(QrcpArgs<double2> a) {
    __shared__ double2 red[QP_THREADS / 32][QP_GCOLS<double2>];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t j = a.j;
    const int64_t c0 = a.k0 + (int64_t)blockIdx.x * QP_GCOLS<double2>;
    const int64_t r0 = j + (int64_t)blockIdx.y * a.split_rows, r1 = min(a.m, r0 + a.split_rows);
    const int ncl = (int)min((int64_t)QP_GCOLS<double2>, a.n - c0);
    const double2* A0 = a.A + c0 * a.lda;
    double re[QP_GCOLS<double2>], im[QP_GCOLS<double2>];
#pragma unroll
    for (int q = 0; q < QP_GCOLS<double2>; ++q) { re[q] = 0.0; im[q] = 0.0; }
    if (ncl == QP_GCOLS<double2> && (j < c0 || j >= c0 + QP_GCOLS<double2>)) {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double2 xi = a.x[i - j];
            double2 v[QP_GCOLS<double2>];
#pragma unroll
            for (int q = 0; q < QP_GCOLS<double2>; ++q) v[q] = A0[(int64_t)q * a.lda + i];
#pragma unroll
            for (int q = 0; q < QP_GCOLS<double2>; ++q) {
                re[q] += v[q].x * xi.x + v[q].y * xi.y;
                im[q] += v[q].x * xi.y - v[q].y * xi.x;
            }
        }
    } else {
        for (int64_t i = r0 + tid; i < r1; i += QP_THREADS) {
            const double2 xi = a.x[i - j];
#pragma unroll
            for (int q = 0; q < QP_GCOLS<double2>; ++q)
                if (q < ncl && c0 + q != j) {
                    const double2 v = A0[(int64_t)q * a.lda + i];
                    re[q] += v.x * xi.x + v.y * xi.y;
                    im[q] += v.x * xi.y - v.y * xi.x;
                }
        }
    }
#pragma unroll
    for (int q = 0; q < QP_GCOLS<double2>; ++q) {
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
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_finish(QrcpArgs<double2> a) {
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
template <typename T>
__global__ void __launch_bounds__(QP_THREADS) k_qrcp_renorm(QrcpArgs<T> a) {
    __shared__ T sF[QP_NB];
    __shared__ double red[QP_THREADS / 32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nl = a.jj + 1;
    const T* Ak = a.A + a.k0 * a.lda;
    for (int64_t c = a.j + 1 + blockIdx.x; c < a.n; c += gridDim.x) {
        if (!a.flag[c]) continue;
        __syncthreads();
        if (tid < nl) sF[tid] = a.F[c + tid * a.ldf];
        __syncthreads();
        const T* col = a.A + c * a.lda;
        double s = 0.0;
        for (int64_t i = a.j + 1 + tid; i < a.m; i += QP_THREADS) {
            T v = col[i];
            for (int l = 0; l < nl; ++l) v -= qp_mul_conj(Ak[(int64_t)l * a.lda + i], sF[l]);
            s += qp_abs2(v);
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

// Y^ of one complex panel in the ypk layout of the 128-instantiation of C += V Y (nkq_alloc = 4 k-chunks per column tile, the
// first two written: real k index kk = 2l + (0: real part, 1: imaginary part) of reflector l): Y^[2l, c] = -Re F[c0 + c, l],
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
template <typename T>
__global__ void k_qrcp_scatter(const T* __restrict__ z, int64_t ldz, const int64_t* __restrict__ jpvt, int64_t n, int64_t rank,
                               T* __restrict__ b, int64_t ldb) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t d = jpvt[i];
    if (d < 0 || d >= n) return;
    b[d + (int64_t)blockIdx.y * ldb] = i < rank ? z[i + (int64_t)blockIdx.y * ldz] : zero<T>();
}

// Complete orthogonal decomposition (dhqr_cod_*): F (n x rank) <- R_r^H, R_r = rows [0, rank) of R = triu(A, 1) + diag(alpha), so
// F[j, i] = conj(A[i, j]) for j > i, conj(alpha[i]) for j = i and 0 for j < i.  One CTA per 32 x 32 tile of F: the strip of A it
// needs is read along A's columns (coalesced), transposed through shared memory and written along F's columns.  A tile that lies
// wholly above F's diagonal is zero and reads nothing; the strict lower triangle of A (the reflectors) is never read.
constexpr int CP_TILE = 32, CP_ROWS = 8;
template <typename T>
__global__ void __launch_bounds__(CP_TILE * CP_ROWS) k_cod_pack(const T* __restrict__ A, int64_t lda, const T* __restrict__ alpha,
                                                                int64_t n, int64_t rank, T* __restrict__ F, int64_t ldf) {
    __shared__ T t[CP_TILE][CP_TILE + 1];                              // t[j - j0][i - i0]
    const int64_t j0 = (int64_t)blockIdx.x * CP_TILE, i0 = (int64_t)blockIdx.y * CP_TILE;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const bool lower = j0 + CP_TILE - 1 >= i0;                         // the tile holds some j >= i
    if (lower) {
        for (int r = ty; r < CP_TILE; r += CP_ROWS) {
            const int64_t j = j0 + r, i = i0 + tx;                     // row i of column j of A
            t[r][tx] = qp_rrh(A, lda, alpha, n, rank, i, j);
        }
        __syncthreads();
    }
    for (int r = ty; r < CP_TILE; r += CP_ROWS) {
        const int64_t i = i0 + r, j = j0 + tx;                         // row j of column i of F
        if (i < rank && j < n) F[j + i * ldf] = lower ? t[tx][r] : zero<T>();
    }
}

}  // namespace dhqr
