// dhqr_append.cuh — triangular-pentagonal QR on the device (LAPACK dtpqrt / dtpmqrt): fold k new rows B into the n x n triangle R
// of an existing factorisation, [R; B] = Q~ [R'; 0], DESIGN §2.10; and its hyperbolic twin, the downdate (HYP = true, DESIGN §2.11):
// delete k rows Z, Theta [R; Z] = [R'; 0] with R''R' = R'R - Z'Z and Theta J-orthogonal for J = diag(I_n, -I_k).
//
// Reflector j is H~_j = I - v~_j v~_j' with v~_j = vtop[j] on row j of the R block and B[:, j] (overwritten) on the k new rows; no
// other row of the R block is touched, so row j of R is changed by reflector j alone.  The blocked driver in dhqr_api.cu runs the
// bulk of the work (W = V2' B, C += V2 Y) through the existing DMMA kernels on B with V = V2 (the reflector tails); the three kernels
// here add what the vtop rows bring:
//   k_tp_panel  factors one 32-column panel of [R; B] (the B slab resident in shared memory, the panel's 32 x 32 triangle of R in
//               every CTA), one grid-wide exchange per column, and writes V2 into the packed V buffer for the GEMMs;
//   k_tp_wpart  writes diag(vtop) R[rows, trail] as one more split-K partial of W, so the fixed-order reduction adds it;
//   k_tp_rows   R[rows, trail] += diag(vtop) Y, Y read from the packed ypk layout.
// The downdate's reflector is Theta_j = I - v~_j v~_j' J (v~'Jv~ = vtop^2 - ||V2||^2 = 2); against the append it flips the sign of
// the B Gram terms twice: inside the column's norm and w (k_tp_panel<true>), and in W and T of the block form (k_tp_wpart<true>,
// k_tinv / k_ymake / k_mid32 with HYP = true).  Every other kernel of the sequence is shared unchanged.
#pragma once
#include "dhqr_kernels.cuh"

namespace dhqr {

struct TpPanelArgs {
    double* B;            // first panel column of B (k rows)
    int64_t ldb;
    int64_t k;            // rows of B
    double* R;            // R[j0, j0]: the panel's triangle (strict upper part read and written; the diagonal is in alpha)
    int64_t ldr;
    double* alpha;        // alpha[0:ncols]: diag(R) on entry, diag(R') on return
    double* vtop;         // vtop[0:ncols]
    int ncols;            // active columns (<= IB)
    double* vpk;          // packed V2 of the outer panel
    int voff;             // first packed column of this panel
    int64_t vrows;        // window rows incl. padding (rows >= k are zero-filled)
    int rows_per_cta;
    int lds;              // slab leading dimension
    unsigned long long* cells;   // exchange cells, the k_panel layout: [IB steps][(G + 2) * IB cells][2 words]
    uint32_t epoch;       // tags epoch+1 .. epoch+IB belong to this launch
    int64_t* info;        // downdate only: 0, or the 1-based column that failed (read at launch start, written by CTA 0)
    int64_t col0;         // downdate only: global index of the panel's first column
};

// One column j of the stacked panel x = [R[j, j]; B[:, j]] per step (R's rows below j in the panel are zero and stay zero):
//   every CTA publishes its partials of B[:, j]' B[:, c] (c >= j); the owner warp of column c (CTA c % G) sums the G partials in
//   CTA order and publishes the total; every CTA then forms, from identical data,
//   s = sqrt(t_jj + x0^2), alpha = -sign(x0) s (a zero x0 counts as positive), f = 1 / sqrt(s (s + |x0|)),
//   vtop = f (x0 - alpha), v_B = f B[:, j], and w_c = v~' a_c = f t_jc + vtop R[j, c];
//   then B[:, c] -= v_B w_c in its slab and R[j, c] -= vtop w_c in its copy of the triangle.  s = 0 stores v = 0 and alpha = 0.
// HYP (the downdate, B = Z): s^2 = (|x0| - sqrt(t_jj)) (|x0| + sqrt(t_jj)), w_c = vtop R[j, c] - f t_jc, otherwise the same.  The
// first column with s^2 <= 0 while t_jj > 0, or a NaN s^2, fails: CTA 0 writes its 1-based global index to *info, and from it on
// (and in every later launch, which finds *info != 0 at its start) the columns store vtop = 0, V2 = 0, alpha = NaN, so Theta_j = I.
// Every CTA decides from identical data (the exchanged totals and its own copy of the triangle).
template <bool HYP>
__global__ void __launch_bounds__(PANEL_THREADS, 1) k_tp_panel(TpPanelArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* S = reinterpret_cast<double*>(smem_raw);   // [IB][lds]
    __shared__ double Rt[IB][IB + 1];                   // Rt[i][c] = R[i, c] of the panel, i <= c
    __shared__ double tot[IB], w[IB];
    __shared__ double sc[3];                            // f, vtop, alpha of the column in flight
    __shared__ int dead, first;                         // HYP: a column failed (here or earlier); this launch's first failure

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = gridDim.x, cta = blockIdx.x;
    const int64_t row0 = (int64_t)cta * a.rows_per_cta;
    const int nr = (int)max((int64_t)0, min((int64_t)a.rows_per_cta, a.k - row0));
    const int lds = a.lds, nc = a.ncols;
    const size_t step_words = ((size_t)G * IB + 2 * IB) * 2;
    auto pcell = [&](int step, int g, int c) { return a.cells + (size_t)step * step_words + ((size_t)g * IB + c) * 2; };
    auto tcell = [&](int step, int c) { return a.cells + (size_t)step * step_words + ((size_t)G * IB + c) * 2; };

    for (int c = warp; c < nc; c += PNW)
        for (int r = lane; r < nr; r += 32) S[c * lds + r] = a.B[(int64_t)c * a.ldb + row0 + r];
    for (int e = tid; e < IB * IB; e += PANEL_THREADS) {
        const int i = e % IB, c = e / IB;
        Rt[i][c] = (i < nc && c < nc && i <= c) ? (i == c ? a.alpha[i] : a.R[(int64_t)c * a.ldr + i]) : 0.0;
    }
    if constexpr (HYP) {   // read before this CTA publishes anything, so before CTA 0 can write *info in this launch
        if (tid == 0) { dead = __ldcg(a.info) != 0; first = -1; }
    }
    __syncthreads();

    for (int j = 0; j < nc; ++j) {
        const uint32_t tag = a.epoch + 1 + j;
        // partial dots of column j against columns c >= j, then the owner gather (fixed order: lane l sums CTAs l, l+32, ...)
        for (int c = j + warp; c < nc; c += PNW) {
            double acc = 0.0;
            for (int r = lane; r < nr; r += 32) acc += S[j * lds + r] * S[c * lds + r];
            acc = warp_sum(acc);
            if (lane == 0) ll_store(pcell(j, cta, c), acc, tag);
            if (c % G != cta) continue;
            unsigned long long w0[PANEL_MAXG / 32], w1[PANEL_MAXG / 32];
#pragma unroll
            for (int t = 0; t < PANEL_MAXG / 32; ++t)
                if (lane + 32 * t < G) ll_peek(pcell(j, lane + 32 * t, c), w0[t], w1[t]);
            double sum = 0.0;
#pragma unroll
            for (int t = 0; t < PANEL_MAXG / 32; ++t)
                if (lane + 32 * t < G) sum += ll_finish(pcell(j, lane + 32 * t, c), w0[t], w1[t], tag);
            sum = warp_sum(sum);
            if (lane == 0) ll_store(tcell(j, c), sum, tag);
        }
        if (warp == 0 && lane >= j && lane < nc) tot[lane] = ll_wait(tcell(j, lane), tag);
        __syncthreads();
        if (warp == 0) {
            const double x0 = Rt[j][j];
            if constexpr (!HYP) {
                const double s = sqrt(tot[j] + x0 * x0);
                const double alpha = s == 0.0 ? 0.0 : (x0 >= 0.0 ? -s : s);
                const double f = s == 0.0 ? 0.0 : 1.0 / sqrt(s * (s + fabs(x0)));
                const double vt = f * (x0 - alpha);
                if (lane > j && lane < nc) {
                    const double wc = f * tot[lane] + vt * Rt[j][lane];
                    w[lane] = wc;
                    Rt[j][lane] -= vt * wc;
                }
                if (lane == 0) {
                    sc[0] = f; sc[1] = vt; sc[2] = alpha;
                    Rt[j][j] = alpha;
                }
            } else {
                const double t = tot[j], ax = fabs(x0), rt = sqrt(t);
                const double s2 = (ax - rt) * (ax + rt);
                const bool fails = isnan(s2) || (t > 0.0 && s2 <= 0.0);
                const bool off = dead || fails;
                __syncwarp();
                const double s = off ? 0.0 : sqrt(s2);
                const double alpha = off ? __longlong_as_double(0x7ff8000000000000ll) : (s == 0.0 ? 0.0 : (x0 >= 0.0 ? -s : s));
                const double f = (off || s == 0.0) ? 0.0 : 1.0 / sqrt(s * (s + ax));
                const double vt = off ? 0.0 : f * (x0 - alpha);
                if (lane > j && lane < nc) {
                    const double wc = off ? 0.0 : vt * Rt[j][lane] - f * tot[lane];
                    w[lane] = wc;
                    Rt[j][lane] -= vt * wc;
                }
                if (lane == 0) {
                    sc[0] = f; sc[1] = vt; sc[2] = alpha;
                    Rt[j][j] = alpha;
                    if (off && !dead) { dead = 1; first = j; }
                }
            }
        }
        __syncthreads();
        const double f = sc[0];
        const bool zero_v = HYP && dead;   // HYP: column j is off (dead only turns on), V2 = +0 exactly
        for (int r = tid; r < nr; r += PANEL_THREADS) {
            const double v = zero_v ? 0.0 : f * S[j * lds + r];
            S[j * lds + r] = v;
            for (int c = j + 1; c < nc; ++c) S[c * lds + r] -= v * w[c];
        }
        if (cta == 0 && tid == 0) { a.alpha[j] = sc[2]; a.vtop[j] = sc[1]; }
        __syncthreads();
    }
    if constexpr (HYP) {
        if (cta == 0 && tid == 0 && first >= 0) a.info[0] = a.col0 + first + 1;
    }

    for (int c = warp; c < nc; c += PNW)
        for (int r = lane; r < nr; r += 32) a.B[(int64_t)c * a.ldb + row0 + r] = S[c * lds + r];
    if (cta == 0)
        for (int e = tid; e < IB * IB; e += PANEL_THREADS) {
            const int i = e % IB, c = e / IB;
            if (i < c && c < nc) a.R[(int64_t)c * a.ldr + i] = Rt[i][c];
        }
    for (int c = warp; c < IB; c += PNW) {
        const int pc = a.voff + c;
        for (int r = lane; r < nr; r += 32) a.vpk[vpk_index(row0 + r, pc)] = c < nc ? S[c * lds + r] : 0.0;
        if (cta == G - 1)
            for (int64_t r = a.k + lane; r < a.vrows; r += 32) a.vpk[vpk_index(r, pc)] = 0.0;
    }
}

// The vtop rows' share of W = V~' C as split-K partial `Wp` ([next][nbpk] column-major, next = nv + ncols): zero in the nv Gram
// columns (each vtop sits on its own row, so V~'V~ and V2'V2 agree off the diagonal), vtop[i] * X[i, col] in W column col, where X
// (rows [0, kb), ncols columns, ldx) is the block's rows of R (or of c in the apply functions).  Rows kb..nbpk-1 are zero.
// HYP (the downdate) writes -vtop[i] * X[i, col]: the reduced W columns are then V2'C - diag(vtop) X = -(V~'J [X; C]).
template <bool HYP>
__global__ void k_tp_wpart(double* __restrict__ Wp, int nbpk, int nv, int ncols, const double* __restrict__ vtop, int kb,
                           const double* __restrict__ X, int64_t ldx) {
    const int64_t nelem = (int64_t)(nv + ncols) * nbpk;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nelem; e += (int64_t)gridDim.x * blockDim.x) {
        const int col = (int)(e / nbpk) - nv, i = (int)(e % nbpk);
        const double p = (col >= 0 && i < kb) ? vtop[i] * X[(int64_t)col * ldx + i] : 0.0;
        Wp[e] = HYP ? -p : p;
    }
}

// X[i, col] += vtop[i] * Y[i, col], i < kb, col < ncols: the vtop rows' share of C += V~ Y.  Y = -T'W (or -TW) in the ypk layout
// of k_ymake / k_mid32 with nkq = nbpk / KC k-chunks per column tile.
__global__ void k_tp_rows(double* __restrict__ X, int64_t ldx, int ncols, const double* __restrict__ vtop, int kb,
                          const double* __restrict__ ypk, int nkq) {
    const int64_t nelem = (int64_t)ncols * kb;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nelem; e += (int64_t)gridDim.x * blockDim.x) {
        const int col = (int)(e / kb), i = (int)(e % kb);
        const double y = ypk[((int64_t)(col / YT) * nkq + i / KC) * (YT * LDK) + (col % YT) * LDK + (i % KC)];
        X[(int64_t)col * ldx + i] += vtop[i] * y;
    }
}

}  // namespace dhqr
