// dhqr_batched.cuh — batched QR of many small problems and their solves (dhqr_qr_batched_f64, dhqr_apply_qt_batched_f64,
// dhqr_apply_q_batched_f64, dhqr_solve_batched_f64; DESIGN §2.12).
//
// One thread-block cluster per problem (and per chunk of right-hand-side columns for the applies).  CTA `r` of a cluster of `cs`
// holds rows [r * rpc, min(m, (r + 1) * rpc)) of its problem in shared memory for the whole launch.  Every reduction runs in a
// fixed order that depends on (m, n) only: per-thread strided sums, a xor-shuffle tree within the warp, the warp partials in warp
// order, then the CTA partials in rank order, read by every CTA through distributed shared memory.  So every CTA of a cluster holds
// the same total, and the bits of a problem's result depend on its own data and shape only: not on its position in the batch,
// the leading dimensions, the strides or the base address.  The arithmetic is the reference's column step (S:127-135, S:208-209)
// on FP64 CUDA cores; nothing is written outside the operands, and there is no workspace.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

constexpr int BQ_SLAB = 24576;                                    // doubles one CTA's slab is sized for (192 KiB)
constexpr int BQ_MAX_CLUSTER = 8;                                 // portable cluster size limit
constexpr int64_t BQ_MAX_ELEMS = (int64_t)BQ_MAX_CLUSTER * BQ_SLAB;  // the size limit m * n (read-only option batch_max_elems)
constexpr int BQ_KC = 32;                                         // right-hand-side columns per chunk, at most

// The launch geometry of a problem shape.  A function of (m, n) only, so it fixes every summation order.
struct BatchedGeom {
    int cs;        // CTAs per cluster: the smallest of 1, 2, 4, 8 whose row slabs of n columns fit BQ_SLAB (8 above that)
    int rpc;       // rows per CTA, ceil(m / cs); at cs = 8 and m * n <= BQ_MAX_ELEMS a slab holds < BQ_SLAB + n doubles
    int threads;   // 32 per warp, as many warps as the slab has 32-row groups or columns (at least 1, at most 8)
};

__host__ __device__ inline BatchedGeom batched_geom(int64_t m, int64_t n) {
    BatchedGeom g;
    g.cs = 1;
    while (g.cs < BQ_MAX_CLUSTER && ((m + g.cs - 1) / g.cs) * n > BQ_SLAB) g.cs *= 2;
    g.rpc = (int)((m + g.cs - 1) / g.cs);
    const int64_t wr = (g.rpc + 31) / 32, wc = n;
    int64_t w = wr > wc ? wr : wc;
    w = w < 1 ? 1 : (w > 8 ? 8 : w);
    g.threads = 32 * (int)w;
    return g;
}

// right-hand-side columns per chunk of the applies: the b slab and (solve) the gathered top n rows fit BQ_SLAB + n doubles
inline int batched_kc(const BatchedGeom& g, int64_t n, int nrhs) {
    int64_t kc = BQ_SLAB / ((int64_t)g.rpc + n);
    kc = kc < 1 ? 1 : (kc > BQ_KC ? BQ_KC : kc);
    return (int)(kc < nrhs ? kc : nrhs);
}

inline size_t smem_qr_batched(const BatchedGeom& g, int64_t n) { return ((size_t)g.rpc * n + 2 * (size_t)n + 8 + 2) * 8; }
inline size_t smem_apply_batched(const BatchedGeom& g, int64_t n, int kc, bool solve) {
    return ((size_t)g.rpc * kc + (solve ? (size_t)n * kc : 0) + (size_t)kc * (8 + 3)) * 8;
}

__device__ __forceinline__ uint32_t bq_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t bq_nrank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
// Every thread of every CTA of the cluster; orders shared-memory accesses across the cluster (release / acquire).
__device__ __forceinline__ void bq_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// The double at the offset of `p` in CTA `cta` of the cluster.
__device__ __forceinline__ double bq_ld_cluster(const double* p, uint32_t cta) {
    uint32_t remote;
    double v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(cta));
    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(remote) : "memory");
    return v;
}
__device__ __forceinline__ double bq_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// The first local row >= lo that thread `t` of `T` owns: a thread owns the rows i with i % T == t, in every column step, so the
// norm of column j + 1 reads exactly the entries this thread updated in step j.
__device__ __forceinline__ int bq_first(int lo, int t, int T) { return lo <= t ? t : t + (lo - t + T - 1) / T * T; }

// x = R^{-1} xs for kw right-hand sides xs ([kw][n] in shared memory, overwritten) by the block's threads, then x to b[0:n, 0:kw]
// (leading dimension ldb).  R = triu(R, 1) + diag(ap): only the strict upper triangle of R and ap are read.  Column i of R at a
// time, from the last: x_i = xs_i / ap[i], then xs[0:i] -= R[0:i, i] x_i; every entry sees its updates in the order of i, whatever
// the block size.
__device__ __forceinline__ void bq_backsolve(double* xs, int n, int kw, const double* __restrict__ R, int64_t ldr,
                                             const double* __restrict__ ap, double* __restrict__ b, int64_t ldb) {
    const int tid = threadIdx.x, T = blockDim.x;
    for (int i = n - 1; i >= 0; --i) {
        for (int k = tid; k < kw; k += T) xs[(int64_t)k * n + i] /= ap[i];
        __syncthreads();
        const double* Ri = R + (int64_t)i * ldr;
        for (int64_t e = tid; e < (int64_t)i * kw; e += T) {
            const int k = (int)(e / i), l = (int)(e - (int64_t)k * i);
            xs[(int64_t)k * n + l] -= Ri[l] * xs[(int64_t)k * n + i];
        }
        __syncthreads();
    }
    for (int64_t e = tid; e < (int64_t)n * kw; e += T) {
        const int k = (int)(e / n), i = (int)(e - (int64_t)k * n);
        b[(int64_t)k * ldb + i] = xs[(int64_t)k * n + i];
    }
}

// Factor problem blockIdx.x / cs in place.  Per column j: (1) each CTA's partial of ||A[j:, j]||^2; cluster barrier; every CTA sums
// the partials in rank order and reads x0 = A[j, j] from the CTA that holds row j; (2) alpha, f and v in place (S:129-135, sign(0)
// = 0 as in the reference); (3) w_c = v' A[j:, c] for c > j, warps owning columns and lanes rows; cluster barrier; every CTA sums
// the w partials in rank order; (4) A[j:, c] -= v w_c on the slab.  Single buffers suffice: a partial of step j + 1 is written only
// after the barrier that every CTA reaches after reading the step-j value it replaces.  No CTA reads another's shared memory after
// the second barrier of the last column, so none needs to wait for the others before it exits.
__global__ void __launch_bounds__(256) k_qr_batched(double* __restrict__ A, int64_t lda, int64_t stride_a, double* __restrict__ alpha,
                                                    int64_t stride_alpha, int m, int n, int rpc) {
    extern __shared__ double bq_sm[];
    double* red = bq_sm;               // [8] warp partials
    double* part = red + 8;            // [1] this CTA's norm partial
    double* xj = part + 1;             // [1] x0, in the CTA that holds row j
    double* wpart = xj + 1;            // [n] this CTA's partials of w
    double* wsum = wpart + n;          // [n] w
    double* S = wsum + n;              // [n][rpc] the slab, column-major
    const int tid = threadIdx.x, T = blockDim.x, warp = tid >> 5, lane = tid & 31, nw = T >> 5;
    const uint32_t cs = bq_nrank(), rank = bq_rank();
    const int64_t prob = blockIdx.x / cs;
    double* Ap = A + prob * stride_a;
    double* al = alpha + prob * stride_alpha;
    const int r0 = (int)rank * rpc;
    const int nr = max(0, min(m - r0, rpc));

    for (int64_t e = tid; e < (int64_t)nr * n; e += T) {
        const int c = (int)(e / nr), i = (int)(e - (int64_t)c * nr);
        S[(int64_t)c * rpc + i] = Ap[(int64_t)c * lda + r0 + i];
    }
    __syncthreads();

    for (int j = 0; j < n; ++j) {
        const int lo = max(j - r0, 0);
        const double* Sj = S + (int64_t)j * rpc;
        double acc = 0.0;
        for (int i = bq_first(lo, tid, T); i < nr; i += T) acc += Sj[i] * Sj[i];
        acc = bq_warp_sum(acc);
        if (lane == 0) red[warp] = acc;
        __syncthreads();
        if (tid == 0) {
            double p = 0.0;
            for (int w = 0; w < nw; ++w) p += red[w];
            part[0] = p;
            if (j >= r0 && j < r0 + nr) xj[0] = Sj[j - r0];
        }
        bq_cluster_sync();
        double t = 0.0;
        for (uint32_t q = 0; q < cs; ++q) t += bq_ld_cluster(part, q);
        const double x0 = bq_ld_cluster(xj, (uint32_t)(j / rpc));
        const double s = sqrt(t);                                               // S:129
        const double sg = x0 > 0.0 ? 1.0 : (x0 < 0.0 ? -1.0 : 0.0);
        const double a = -sg * s;                                               // S:130
        const double f = 1.0 / sqrt(s * (s + fabs(x0)));                        // S:131
        for (int i = bq_first(lo, tid, T); i < nr; i += T) {                    // S:132-135
            double x = Sj[i];
            if (r0 + i == j) x -= a;
            S[(int64_t)j * rpc + i] = x * f;
        }
        if (tid == 0 && j >= r0 && j < r0 + nr) al[j] = a;
        __syncthreads();
        for (int c = j + 1 + warp; c < n; c += nw) {                            // S:208
            const double* Sc = S + (int64_t)c * rpc;
            double w = 0.0;
            for (int i = lo + lane; i < nr; i += 32) w += Sj[i] * Sc[i];
            w = bq_warp_sum(w);
            if (lane == 0) wpart[c] = w;
        }
        bq_cluster_sync();
        for (int c = j + 1 + tid; c < n; c += T) {
            double w = 0.0;
            for (uint32_t q = 0; q < cs; ++q) w += bq_ld_cluster(wpart + c, q);
            wsum[c] = w;
        }
        __syncthreads();
        for (int i = bq_first(lo, tid, T); i < nr; i += T) {                    // S:209
            const double v = Sj[i];
            for (int c = j + 1; c < n; ++c) S[(int64_t)c * rpc + i] -= v * wsum[c];
        }
    }
    __syncthreads();
    for (int64_t e = tid; e < (int64_t)nr * n; e += T) {
        const int c = (int)(e / nr), i = (int)(e - (int64_t)c * nr);
        Ap[(int64_t)c * lda + r0 + i] = S[(int64_t)c * rpc + i];
    }
}

// b <- Q'b (TRANS) or Q b of problem blockIdx.x / cs, for right-hand-side chunks blockIdx.y, blockIdx.y + gridDim.y, ... of kc
// columns held in shared memory with the row split of k_qr_batched.  Reflector j is read from global memory, each CTA its own
// rows.  Per reflector: the partials of w_k = v' b_k (threads own rows, as in the norm of k_qr_batched), one cluster barrier, the
// sums in rank order, b_k -= v w_k.  The w partials alternate between two buffers, so the one written for a reflector is never the
// one another CTA may still be reading for the previous reflector.  SOLVE (with TRANS): after the sweep CTA 0 gathers (Q'b)[0:n]
// through distributed shared memory and back-substitutes with R = triu(A, 1) + diag(alpha) read from global memory, column by
// column in a fixed order; b[0:n] <- x, rows n..m-1 keep (Q'b)[n:m].
template <bool TRANS, bool SOLVE>
__global__ void __launch_bounds__(256) k_apply_batched(const double* __restrict__ A, int64_t lda, int64_t stride_a,
                                                       const double* __restrict__ alpha, int64_t stride_alpha, double* __restrict__ b,
                                                       int64_t ldb, int64_t stride_b, int m, int n, int nrhs, int rpc, int kc) {
    extern __shared__ double bq_sm[];
    double* red = bq_sm;               // [kc][8] warp partials
    double* wpart = red + 8 * kc;      // [2][kc] this CTA's partials of w
    double* wsum = wpart + 2 * kc;     // [kc] w
    double* Bs = wsum + kc;            // [kc][rpc] the b slab
    double* xs = Bs + (int64_t)kc * rpc;   // [kc][n] (SOLVE, CTA 0) the gathered top n rows, then x
    const int tid = threadIdx.x, T = blockDim.x, warp = tid >> 5, lane = tid & 31, nw = T >> 5;
    const uint32_t cs = bq_nrank(), rank = bq_rank();
    const int64_t prob = blockIdx.x / cs;
    const double* Ap = A + prob * stride_a;
    double* bp = b + prob * stride_b;
    const int r0 = (int)rank * rpc;
    const int nr = max(0, min(m - r0, rpc));
    int it = 0;

    for (int k0 = blockIdx.y * kc; k0 < nrhs; k0 += gridDim.y * kc) {
        const int kw = min(kc, nrhs - k0);
        for (int64_t e = tid; e < (int64_t)nr * kw; e += T) {
            const int k = (int)(e / nr), i = (int)(e - (int64_t)k * nr);
            Bs[(int64_t)k * rpc + i] = bp[(int64_t)(k0 + k) * ldb + r0 + i];
        }
        __syncthreads();
        for (int jj = 0; jj < n; ++jj, ++it) {
            const int j = TRANS ? jj : n - 1 - jj;
            const int lo = max(j - r0, 0);
            const double* v = Ap + (int64_t)j * lda + r0;
            double* wp = wpart + (it & 1) * kc;
            for (int k = 0; k < kw; ++k) {
                const double* Bk = Bs + (int64_t)k * rpc;
                double acc = 0.0;
                for (int i = bq_first(lo, tid, T); i < nr; i += T) acc += v[i] * Bk[i];
                acc = bq_warp_sum(acc);
                if (lane == 0) red[k * 8 + warp] = acc;
            }
            __syncthreads();
            for (int k = tid; k < kw; k += T) {
                double p = 0.0;
                for (int w = 0; w < nw; ++w) p += red[k * 8 + w];
                wp[k] = p;
            }
            bq_cluster_sync();
            for (int k = tid; k < kw; k += T) {
                double w = 0.0;
                for (uint32_t q = 0; q < cs; ++q) w += bq_ld_cluster(wp + k, q);
                wsum[k] = w;
            }
            __syncthreads();
            for (int i = bq_first(lo, tid, T); i < nr; i += T) {
                const double vi = v[i];
                for (int k = 0; k < kw; ++k) Bs[(int64_t)k * rpc + i] -= vi * wsum[k];
            }
        }
        if constexpr (SOLVE) {
            bq_cluster_sync();                                                  // every CTA's rows are final
            if (rank == 0) {
                for (int64_t e = tid; e < (int64_t)n * kw; e += T) {
                    const int k = (int)(e / n), i = (int)(e - (int64_t)k * n);
                    const uint32_t q = (uint32_t)(i / rpc);
                    xs[(int64_t)k * n + i] = bq_ld_cluster(Bs + (int64_t)k * rpc + (i - (int)q * rpc), q);
                }
            }
            const int ilo = max(n - r0, 0);                                     // rows n..m-1: (Q'b)[n:m]
            for (int64_t e = tid; e < (int64_t)max(nr - ilo, 0) * kw; e += T) {
                const int k = (int)(e / (nr - ilo)), i = ilo + (int)(e - (int64_t)k * (nr - ilo));
                bp[(int64_t)(k0 + k) * ldb + r0 + i] = Bs[(int64_t)k * rpc + i];
            }
            bq_cluster_sync();                                                  // CTA 0 has read every slab
            if (rank == 0) bq_backsolve(xs, n, kw, Ap, lda, alpha + prob * stride_alpha, bp + (int64_t)k0 * ldb, ldb);
        } else {
            __syncthreads();
            for (int64_t e = tid; e < (int64_t)nr * kw; e += T) {
                const int k = (int)(e / nr), i = (int)(e - (int64_t)k * nr);
                bp[(int64_t)(k0 + k) * ldb + r0 + i] = Bs[(int64_t)k * rpc + i];
            }
        }
        __syncthreads();
    }
    bq_cluster_sync();   // no CTA leaves while another may still read its w partials
}

// ---- batched append and downdate (dhqr_qr_append_batched_f64, dhqr_qr_downdate_batched_f64; DESIGN §2.13) ---------------------
// Problem i folds its k x n block B (or removes Z) into its n x n triangle R, and transforms [c; e] with the same reflectors: the
// column steps of k_tp_panel (dhqr_append.cuh) on one problem per cluster.  The slab of CTA r is rows [r * rpc, (r + 1) * rpc) of
// [B | e], n + nrhs columns, column-major; the geometry is batched_geom(k, n + nrhs).  R is never held: row j of R and of c is read
// from global memory at step j, and only reflector j touches it.
constexpr int BQ_UPD_MAX_COLS = 1024;   // n + nrhs at most (read-only option batch_update_max_cols); k (n + nrhs) <= BQ_MAX_ELEMS
// Shared memory: the slab and three column vectors.  At cs = 8, rpc (n + nrhs) < BQ_SLAB + (n + nrhs), so the worst case is
// (24 576 + 4 x 1024) x 8 B = 229 376 B, inside the 227 KiB (232 448 B) a CTA may opt in to.
inline size_t smem_tp_batched(const BatchedGeom& g, int64_t ncol) { return ((size_t)g.rpc * ncol + 3 * (size_t)ncol) * 8; }

// Per column j, with x0 = alpha[j] and R[j, :] as they are on entry (reflectors 0..j-1 never touch row j):
//   (1) each warp owns columns c >= j of the slab and writes this CTA's partial of B[:, j]' B[:, c] (lanes own rows); cluster
//       barrier; every CTA sums the partials in rank order: w[j] = t = ||B[:, j]||^2, w[c] = t_jc;
//   (2) every thread forms, from identical data, the scalars of k_tp_panel: append s = sqrt(t + x0^2), alpha = -sign(x0) s (a zero
//       x0 counts as positive), f = 1 / sqrt(s (s + |x0|)), vtop = f (x0 - alpha), w_c = f t_jc + vtop R[j, c]; downdate s^2 =
//       (|x0| - sqrt(t)) (|x0| + sqrt(t)), w_c = vtop R[j, c] - f t_jc, and the failure rule of dhqr_qr_downdate_f64;
//   (3) B[:, j] <- V2 = f B[:, j], B[:, c] -= V2 w_c on the slab.
// Columns c >= n are the right-hand sides: R[j, c] is then c[j, c - n], and e is transformed with B.  R's row j, c's row j and
// alpha[j] are read by every CTA after the barrier of step j, so CTA 0 writes them (R[j, c] - vtop w_c) after the barrier of step
// j + 1, when no CTA can still read them; the w partials alternate between two buffers for the same reason as in k_apply_batched.
template <bool HYP>
__global__ void __launch_bounds__(256) k_tp_batched(double* __restrict__ R, int64_t ldr, int64_t stride_r, double* __restrict__ alpha,
                                                    int64_t stride_alpha, double* __restrict__ B, int64_t ldb, int64_t stride_b,
                                                    double* __restrict__ vtop, int64_t stride_vtop, double* __restrict__ cm, int64_t ldc,
                                                    int64_t stride_c, double* __restrict__ e, int64_t lde, int64_t stride_e,
                                                    int64_t* __restrict__ info, int n, int k, int nrhs, int rpc) {
    extern __shared__ double bq_sm[];
    const int ncol = n + nrhs;
    double* wpart = bq_sm;               // [2][ncol] this CTA's partials
    double* w = wpart + 2 * ncol;        // [ncol] t_jc, then w_c
    double* S = w + ncol;                // [ncol][rpc] the slab of [B | e]
    const int tid = threadIdx.x, T = blockDim.x, warp = tid >> 5, lane = tid & 31, nw = T >> 5;
    const uint32_t cs = bq_nrank(), rank = bq_rank();
    const int64_t prob = blockIdx.x / cs;
    double* Rp = R + prob * stride_r;
    double* al = alpha + prob * stride_alpha;
    double* Bp = B + prob * stride_b;
    double* cp = cm + prob * stride_c;
    double* ep = e + prob * stride_e;
    const int r0 = (int)rank * rpc;
    const int nr = max(0, min(k - r0, rpc));
    // column c of [R | c] at row j
    auto top = [&](int j, int c) -> double* { return c < n ? Rp + (int64_t)c * ldr + j : cp + (int64_t)(c - n) * ldc + j; };

    for (int64_t x = tid; x < (int64_t)nr * ncol; x += T) {
        const int c = (int)(x / nr), i = (int)(x - (int64_t)c * nr);
        S[(int64_t)c * rpc + i] = c < n ? Bp[(int64_t)c * ldb + r0 + i] : ep[(int64_t)(c - n) * lde + r0 + i];
    }
    __syncthreads();

    double vt_prev = 0.0, a_prev = 0.0;
    bool dead = false;
    int first = -1;
    for (int j = 0; j < n; ++j) {
        const double* Sj = S + (int64_t)j * rpc;
        double* wp = wpart + (j & 1) * ncol;
        for (int c = j + warp; c < ncol; c += nw) {
            const double* Sc = S + (int64_t)c * rpc;
            double acc = 0.0;
            for (int i = lane; i < nr; i += 32) acc += Sj[i] * Sc[i];
            acc = bq_warp_sum(acc);
            if (lane == 0) wp[c] = acc;
        }
        bq_cluster_sync();
        for (int c = j + tid; c < ncol; c += T) {
            if (rank == 0 && j > 0) {                                           // row j - 1, now that no CTA reads it
                double* p = top(j - 1, c);
                *p -= vt_prev * w[c];
            }
            double s = 0.0;
            for (uint32_t q = 0; q < cs; ++q) s += bq_ld_cluster(wp + c, q);
            w[c] = s;
        }
        if (rank == 0 && tid == 0 && j > 0) al[j - 1] = a_prev;
        __syncthreads();
        const double x0 = al[j], t = w[j];
        double f, vt, a;
        if constexpr (!HYP) {
            const double s = sqrt(t + x0 * x0);
            a = s == 0.0 ? 0.0 : (x0 >= 0.0 ? -s : s);
            f = s == 0.0 ? 0.0 : 1.0 / sqrt(s * (s + fabs(x0)));
            vt = f * (x0 - a);
        } else {
            const double ax = fabs(x0), rt = sqrt(t);
            const double s2 = (ax - rt) * (ax + rt);
            const bool fails = isnan(s2) || (t > 0.0 && s2 <= 0.0);
            if (fails && !dead) first = j;
            dead = dead || fails;
            const double s = dead ? 0.0 : sqrt(s2);
            a = dead ? __longlong_as_double(0x7ff8000000000000ll) : (s == 0.0 ? 0.0 : (x0 >= 0.0 ? -s : s));
            f = (dead || s == 0.0) ? 0.0 : 1.0 / sqrt(s * (s + ax));
            vt = dead ? 0.0 : f * (x0 - a);
        }
        for (int c = j + 1 + tid; c < ncol; c += T) {                          // w[j] = t is not overwritten
            const double rc = *top(j, c);
            if constexpr (!HYP) w[c] = f * w[c] + vt * rc;
            else w[c] = dead ? 0.0 : vt * rc - f * w[c];
        }
        if (rank == 0 && tid == 0) vtop[prob * stride_vtop + j] = vt;
        vt_prev = vt;
        a_prev = a;
        __syncthreads();
        for (int i = tid; i < nr; i += T) {
            const double v = (HYP && dead) ? 0.0 : f * Sj[i];
            S[(int64_t)j * rpc + i] = v;
            for (int c = j + 1; c < ncol; ++c) S[(int64_t)c * rpc + i] -= v * w[c];
        }
        __syncthreads();
    }
    bq_cluster_sync();   // no CTA reads row n - 1 or another's partials any more
    if (rank == 0) {
        for (int c = n + tid; c < ncol; c += T) *top(n - 1, c) -= vt_prev * w[c];
        if (tid == 0) {
            al[n - 1] = a_prev;
            if constexpr (HYP) info[prob] = first + 1;
        }
    }
    for (int64_t x = tid; x < (int64_t)nr * ncol; x += T) {
        const int c = (int)(x / nr), i = (int)(x - (int64_t)c * nr);
        const double v = S[(int64_t)c * rpc + i];
        if (c < n) Bp[(int64_t)c * ldb + r0 + i] = v;
        else ep[(int64_t)(c - n) * lde + r0 + i] = v;
    }
}

// b[0:n] <- R^{-1} b[0:n] of problem blockIdx.x for right-hand-side chunks blockIdx.y, blockIdx.y + gridDim.y, ... of kc columns:
// the back-substitution of k_apply_batched<true, true> (bq_backsolve) on b's top n rows, loaded into shared memory.
__global__ void __launch_bounds__(256) k_backsolve_batched(const double* __restrict__ R, int64_t ldr, int64_t stride_r,
                                                           const double* __restrict__ alpha, int64_t stride_alpha, double* __restrict__ b,
                                                           int64_t ldb, int64_t stride_b, int n, int nrhs, int kc) {
    extern __shared__ double bq_sm[];
    double* xs = bq_sm;                  // [kc][n]
    const int tid = threadIdx.x, T = blockDim.x;
    const int64_t prob = blockIdx.x;
    double* bp = b + prob * stride_b;
    for (int k0 = blockIdx.y * kc; k0 < nrhs; k0 += gridDim.y * kc) {
        const int kw = min(kc, nrhs - k0);
        for (int64_t x = tid; x < (int64_t)n * kw; x += T) {
            const int k = (int)(x / n), i = (int)(x - (int64_t)k * n);
            xs[(int64_t)k * n + i] = bp[(int64_t)(k0 + k) * ldb + i];
        }
        __syncthreads();
        bq_backsolve(xs, n, kw, R + prob * stride_r, ldr, alpha + prob * stride_alpha, bp + (int64_t)k0 * ldb, ldb);
        __syncthreads();
    }
}
