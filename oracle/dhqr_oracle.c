/*
 * dhqr_oracle.c — CPU restatement of DistributedHouseholderQR.jl's hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may call into this file.  The product
 * (libdhqr.so) never links, loads or falls back to anything in oracle/.
 *
 * Every function cites the reference lines it follows, with
 *   S:n = line n of the reference's src/DistributedHouseholderQR.jl.
 *
 * Parity status: the reference ships no golden vectors (its tests draw from Julia's
 * Xoshiro stream, test/runtests.jl:6,45-46) and Julia is not installed, so this
 * restatement is pinned by (i) the reference's own test properties (normal-equation
 * residual < 8x LAPACK's, test/runtests.jl:51,62,81; partialdot ~ dot on suffixes,
 * test/partialdot.jl:15-19), (ii) LAPACK dgeqrf through the storage-format identity
 * alpha = diag(R), triu(H,1) = triu(R,1), H[j,j]^2 = tau_j (SURVEY App. A), and
 * (iii) committed fixtures under tests/golden/.  Bitwise parity with the Julia binary
 * is UNPINNED (no Julia here); see DESIGN.md "Oracle".
 *
 * Layout: column-major doubles, leading dimension lda >= m (Julia Matrix / localpart(DArray)).
 * A "column block" is the localpart of the reference's DArray with a (1,P) process grid
 * (test/runtests.jl:71): all m rows of a contiguous global column range (S:33).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define DHQR_ORACLE_VERSION 1

int dhqr_oracle_version(void) { return DHQR_ORACLE_VERSION; }

int dhqr_oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* S:8  alphafactor(x::Real) = -sign(x)   (sign(0) == 0, mirrored on purpose) */
double dhqr_oracle_alphafactor(double x) { return x > 0.0 ? -1.0 : (x < 0.0 ? 1.0 : -0.0 * 0.0); }

/* S:42-49  partialdot(a, b, is, ::Type{<:Real}): sum_{i in is} a[i]*b[i].
 * The reference marks the loop @simd (free re-association); four independent partial
 * sums stand in for the SIMD lanes.  i0..i1 are 0-based, i1 exclusive. */
double dhqr_oracle_partialdot(const double *a, const double *b, int64_t i0, int64_t i1) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    int64_t i = i0;
    for (; i + 4 <= i1; i += 4) {
        s0 += a[i] * b[i];
        s1 += a[i + 1] * b[i + 1];
        s2 += a[i + 2] * b[i + 2];
        s3 += a[i + 3] * b[i + 3];
    }
    for (; i < i1; ++i) s0 += a[i] * b[i];
    return (s0 + s1) + (s2 + s3);
}

/* S:156-160  hotloop!(Hl, Hj, s, is, jj, ::Type{<:Real}): Hl[i,jj] -= Hj[i]*s */
static void hotloop(double *col, const double *hj, double s, int64_t i0, int64_t i1) {
    for (int64_t i = i0; i < i1; ++i) col[i] -= hj[i] * s;
}

/* S:129  norm(view(Hl, j:m, j)) -> LinearAlgebra.norm -> OpenBLAS dnrm2 (OpenBLAS_jll
 * 0.3.23+4, Manifest.toml:139-142; not vendored).  x86-64 OpenBLAS accumulates the squares
 * in extended precision; long double does the same here.  Any faithful 2-norm is within the
 * stated tolerances (parity unpinned at this call boundary, SURVEY 8c). */
static double nrm2(const double *x, int64_t n) {
    long double s = 0.0L;
    for (int64_t i = 0; i < n; ++i) s += (long double)x[i] * (long double)x[i];
    return (double)sqrtl(s);
}

/* A column block: LocalColumnBlock{Al, dj, colrange} of S:26-40.  col0 == dj (0-based first
 * global column), ncols == length(colrange). */
typedef struct {
    double *a;
    int64_t lda;
    int64_t col0;
    int64_t ncols;
} dhqr_oracle_block;

/* S:198-213  _householder_inner!(H, j, Hj): apply (I - v v') to the local columns > j.
 * Columns are split into nthreads contiguous chunks (S:203-205), one thread per chunk
 * (S:206), each column doing partialdot then hotloop! over rows j:m (S:208-209). */
static void householder_inner(const dhqr_oracle_block *blk, int64_t m, int64_t n, int64_t j,
                              const double *hj, int nthreads) {
    int64_t lo = j + 1 > blk->col0 ? j + 1 : blk->col0;           /* intersect(j+1:n, colrange) */
    int64_t hi = blk->col0 + blk->ncols < n ? blk->col0 + blk->ncols : n;
    if (lo >= hi) return;                                          /* S:202 */
    int64_t len = hi - lo;
    int64_t nchunk = (len + nthreads - 1) / nthreads;              /* S:203 */
#pragma omp parallel for schedule(static, 1) num_threads(nthreads)
    for (int t = 0; t < nthreads; ++t) {
        int64_t c0 = lo + (int64_t)t * nchunk;
        int64_t c1 = c0 + nchunk < hi ? c0 + nchunk : hi;
        for (int64_t jj = c0; jj < c1; ++jj) {
            double *col = blk->a + (jj - blk->col0) * blk->lda;
            double s = dhqr_oracle_partialdot(hj, col, j, m);      /* S:208 */
            hotloop(col, hj, s, j, m);                             /* S:209 */
        }
    }
}

/* S:122-148  _householder!(H, alpha) run by the owner of block p, fanning the trailing update out
 * to every block (S:141-143).  S:113-120: owners are visited sequentially in block order. */
int dhqr_oracle_householder_blocks(int64_t m, int64_t n, int nblocks, const dhqr_oracle_block *blocks,
                                   double *alpha, int nthreads) {
    if (m < 0) return -1;
    if (n < 0 || n > m) return -2;
    if (nblocks < 1) return -3;
    if (nthreads < 1) nthreads = dhqr_oracle_max_threads();
    double *hj = (double *)calloc((size_t)(m > 0 ? m : 1), sizeof(double));    /* S:125 */
    if (!hj) return -100;
    for (int p = 0; p < nblocks; ++p) {                            /* S:116 */
        const dhqr_oracle_block *own = &blocks[p];
        for (int64_t j = own->col0; j < own->col0 + own->ncols; ++j) {  /* S:127 */
            double *col = own->a + (j - own->col0) * own->lda;
            double s = nrm2(col + j, m - j);                       /* S:129 */
            alpha[j] = s * dhqr_oracle_alphafactor(col[j]);        /* S:130 */
            double f = 1.0 / sqrt(s * (s + fabs(col[j])));         /* S:131 */
            col[j] -= alpha[j];                                    /* S:132 */
            for (int64_t i = j; i < m; ++i) col[i] *= f;           /* S:133-135 */
            memcpy(hj, col, (size_t)m * sizeof(double));           /* S:138-140 (all m rows) */
            for (int q = 0; q < nblocks; ++q)                      /* S:141-143 */
                householder_inner(&blocks[q], m, n, j, hj, nthreads);
        }
    }
    free(hj);
    return 0;
}

/* S:311-315  qr!(A) for a plain Matrix: one block holding every column. */
int dhqr_oracle_qr(int64_t m, int64_t n, double *a, int64_t lda, double *alpha, int nthreads) {
    if (lda < (m > 1 ? m : 1)) return -4;
    dhqr_oracle_block b = {a, lda, 0, n};
    return dhqr_oracle_householder_blocks(m, n, 1, &b, alpha, nthreads);
}

/* Bounded-sample variant for bench.py's cpu_baseline: runs only column steps [0, jstop) of
 * S:127 on the full matrix and returns the flops those steps performed (S:129-135 + S:208-209
 * counted exactly) through *flops. */
int dhqr_oracle_qr_steps(int64_t m, int64_t n, double *a, int64_t lda, double *alpha, int64_t jstop,
                         int nthreads, double *flops) {
    if (lda < (m > 1 ? m : 1)) return -4;
    if (jstop > n) jstop = n;
    if (nthreads < 1) nthreads = dhqr_oracle_max_threads();
    dhqr_oracle_block b = {a, lda, 0, n};
    double *hj = (double *)calloc((size_t)(m > 0 ? m : 1), sizeof(double));
    if (!hj) return -100;
    double fl = 0.0;
    for (int64_t j = 0; j < jstop; ++j) {
        double *col = a + j * lda;
        double s = nrm2(col + j, m - j);
        alpha[j] = s * dhqr_oracle_alphafactor(col[j]);
        double f = 1.0 / sqrt(s * (s + fabs(col[j])));
        col[j] -= alpha[j];
        for (int64_t i = j; i < m; ++i) col[i] *= f;
        memcpy(hj, col, (size_t)m * sizeof(double));
        householder_inner(&b, m, n, j, hj, nthreads);
        fl += 3.0 * (double)(m - j) + 4.0 * (double)(m - j) * (double)(n - j - 1);
    }
    free(hj);
    if (flops) *flops = fl;
    return 0;
}

/* Strided bounded sample for bench.py: runs the genuine column step of S:127-144 (norm, alpha, scale, copy, trailing
 * update of every column to the right) for j = j0, j0 + stride, j0 + 2 stride, ... < n on whatever the matrix holds.
 * The arithmetic has no data-dependent control flow, so the cost of step j does not depend on the steps before it having
 * run; sampling the whole sweep at a fixed stride covers the early (out-of-cache) and the late (cache-resident) steps in
 * the proportion the full factorisation has them.  *flops = the flops of the sampled steps (counted exactly). */
int dhqr_oracle_qr_steps_strided(int64_t m, int64_t n, double *a, int64_t lda, double *alpha, int64_t j0, int64_t stride,
                                 int nthreads, double *flops) {
    if (lda < (m > 1 ? m : 1)) return -4;
    if (stride < 1 || j0 < 0) return -6;
    if (nthreads < 1) nthreads = dhqr_oracle_max_threads();
    dhqr_oracle_block b = {a, lda, 0, n};
    double *hj = (double *)calloc((size_t)(m > 0 ? m : 1), sizeof(double));
    if (!hj) return -100;
    double fl = 0.0;
    for (int64_t j = j0; j < n; j += stride) {
        double *col = a + j * lda;
        double s = nrm2(col + j, m - j);                           /* S:129 */
        alpha[j] = s * dhqr_oracle_alphafactor(col[j]);            /* S:130 */
        double f = 1.0 / sqrt(s * (s + fabs(col[j])));             /* S:131 */
        col[j] -= alpha[j];                                        /* S:132 */
        for (int64_t i = j; i < m; ++i) col[i] *= f;               /* S:133-135 */
        memcpy(hj, col, (size_t)m * sizeof(double));               /* S:138-140 */
        householder_inner(&b, m, n, j, hj, nthreads);              /* S:141-143 */
        fl += 3.0 * (double)(m - j) + 4.0 * (double)(m - j) * (double)(n - j - 1);
    }
    free(hj);
    if (flops) *flops = fl;
    return 0;
}

/* S:232-242 (and the Vector twin S:215-224)  b <- H_n ... H_1 b = Q'b, owner by owner (S:227-229). */
int dhqr_oracle_apply_qt_blocks(int64_t m, int64_t n, int nblocks, const dhqr_oracle_block *blocks,
                                double *b) {
    for (int p = 0; p < nblocks; ++p) {                            /* S:227 */
        const dhqr_oracle_block *blk = &blocks[p];
        int64_t hi = blk->col0 + blk->ncols < n ? blk->col0 + blk->ncols : n;
        for (int64_t j = blk->col0; j < hi; ++j) {                 /* S:236 */
            const double *col = blk->a + (j - blk->col0) * blk->lda;
            double s = dhqr_oracle_partialdot(col, b, j, m);       /* S:237 */
            for (int64_t i = j; i < m; ++i) b[i] -= col[i] * s;    /* S:238-240 */
        }
    }
    return 0;
}

/* S:272-282  _solve_householder2_inner!: partial row dot over the block's columns > i. */
static double solve2_inner(const dhqr_oracle_block *blk, int64_t n, const double *b, int64_t i) {
    int64_t lo = i + 1 > blk->col0 ? i + 1 : blk->col0;
    int64_t hi = blk->col0 + blk->ncols < n ? blk->col0 + blk->ncols : n;
    double bi = 0.0;                                               /* S:276 */
    for (int64_t j = lo; j < hi; ++j) bi += blk->a[i + (j - blk->col0) * blk->lda] * b[j];  /* S:278-280 */
    return bi;
}

/* S:256-270  back-substitution: for i = n..1, sum the partial dots of every block whose last
 * column is >= i, visiting blocks in reverse order when there is more than one (S:258-259),
 * then b[i] = (b[i] - sum) / alpha[i] (S:266-267). */
int dhqr_oracle_backsolve_blocks(int64_t m, int64_t n, int nblocks, const dhqr_oracle_block *blocks,
                                 const double *alpha, double *b) {
    (void)m;
    for (int64_t i = n - 1; i >= 0; --i) {                         /* S:260 */
        double sum = 0.0;
        for (int q = nblocks - 1; q >= 0; --q) {                   /* S:259, S:262 */
            const dhqr_oracle_block *blk = &blocks[q];
            if (i > blk->col0 + blk->ncols - 1) continue;          /* S:263 */
            sum += solve2_inner(blk, n, b, i);                     /* S:264, S:266 */
        }
        b[i] = (b[i] - sum) / alpha[i];                            /* S:267 */
    }
    return 0;
}

/* S:284-294  solve_householder!(b, H, alpha): Q'b then R^{-1}; x = b[1:n] (S:293). */
int dhqr_oracle_solve_blocks(int64_t m, int64_t n, int nblocks, const dhqr_oracle_block *blocks,
                             const double *alpha, double *b) {
    int rc = dhqr_oracle_apply_qt_blocks(m, n, nblocks, blocks, b);   /* S:288 */
    if (rc) return rc;
    return dhqr_oracle_backsolve_blocks(m, n, nblocks, blocks, alpha, b);  /* S:291 */
}

/* Single-block conveniences (plain Matrix input). */
int dhqr_oracle_apply_qt(int64_t m, int64_t n, const double *a, int64_t lda, double *b) {
    dhqr_oracle_block blk = {(double *)a, lda, 0, n};
    return dhqr_oracle_apply_qt_blocks(m, n, 1, &blk, b);
}
int dhqr_oracle_backsolve(int64_t m, int64_t n, const double *a, int64_t lda, const double *alpha, double *b) {
    dhqr_oracle_block blk = {(double *)a, lda, 0, n};
    return dhqr_oracle_backsolve_blocks(m, n, 1, &blk, alpha, b);
}
/* S:317-321  H \ b: copy b, solve, return the first n entries. */
int dhqr_oracle_ldiv(int64_t m, int64_t n, const double *a, int64_t lda, const double *alpha,
                     const double *b, double *x) {
    double *w = (double *)malloc((size_t)(m > 0 ? m : 1) * sizeof(double));
    if (!w) return -100;
    memcpy(w, b, (size_t)m * sizeof(double));                      /* S:318 */
    dhqr_oracle_block blk = {(double *)a, lda, 0, n};
    int rc = dhqr_oracle_solve_blocks(m, n, 1, &blk, alpha, w);    /* S:319 */
    if (!rc) memcpy(x, w, (size_t)n * sizeof(double));             /* S:320 */
    free(w);
    return rc;
}

/* ---------------------------------------------------------------------------------------------------------------------
 * Extended-precision reference.  The same recurrences as above (S:127-135 column step, S:208-209 trailing update,
 * S:232-242 Q'b sweep, S:256-282 back-substitution, S:317-321 ldiv) carried out in long double and rounded to double only
 * when written out.  Its forward error against exact arithmetic is about kappa * 2^-LDBL_MANT_DIG instead of
 * kappa * 2^-53, so it can measure the fp64 oracle's error and the library's error on the same input, also on inputs
 * where kappa * 1e-16 is large.  Each trailing column is updated by one thread with a sequential sum, so the result does
 * not depend on the thread count.
 * --------------------------------------------------------------------------------------------------------------------- */
typedef long double ldbl;

int dhqr_oracle_ext_mant_dig(void) { return LDBL_MANT_DIG; }

/* S:127-135 + S:208-209 on an m x n long double matrix (leading dimension m) */
static void ext_factor(int64_t m, int64_t n, ldbl *w, ldbl *alpha, int nthreads) {
    for (int64_t j = 0; j < n; ++j) {
        ldbl *col = w + j * m;
        ldbl s = 0.0L;
        for (int64_t i = j; i < m; ++i) s += col[i] * col[i];
        s = sqrtl(s);                                                  /* S:129 */
        const ldbl x = col[j];
        alpha[j] = s * (x > 0.0L ? -1.0L : (x < 0.0L ? 1.0L : -0.0L * 0.0L));   /* S:130, S:8 */
        const ldbl f = 1.0L / sqrtl(s * (s + fabsl(x)));             /* S:131 */
        col[j] -= alpha[j];                                            /* S:132 */
        for (int64_t i = j; i < m; ++i) col[i] *= f;                   /* S:133-135 */
#pragma omp parallel for schedule(static) num_threads(nthreads)
        for (int64_t jj = j + 1; jj < n; ++jj) {
            ldbl *d = w + jj * m;
            ldbl t = 0.0L;
            for (int64_t i = j; i < m; ++i) t += col[i] * d[i];        /* S:208 */
            for (int64_t i = j; i < m; ++i) d[i] -= col[i] * t;        /* S:209 */
        }
    }
}

/* b <- Q'b (S:232-242) or b <- Qb (the same reflectors in reverse order) */
static void ext_apply(int64_t m, int64_t n, const ldbl *w, ldbl *b, int trans) {
    for (int64_t q = 0; q < n; ++q) {
        const int64_t j = trans ? q : n - 1 - q;
        const ldbl *col = w + j * m;
        ldbl s = 0.0L;
        for (int64_t i = j; i < m; ++i) s += col[i] * b[i];           /* S:237 */
        for (int64_t i = j; i < m; ++i) b[i] -= col[i] * s;            /* S:238-240 */
    }
}

/* S:256-282: b[i] = (b[i] - sum_{k>i} R[i,k] b[k]) / alpha[i], i = n..1 */
static void ext_backsolve(int64_t m, int64_t n, const ldbl *w, const ldbl *alpha, ldbl *b) {
    for (int64_t i = n - 1; i >= 0; --i) {
        ldbl sum = 0.0L;
        for (int64_t k = i + 1; k < n; ++k) sum += w[i + k * m] * b[k];
        b[i] = (b[i] - sum) / alpha[i];
    }
}

/* qr!(A) in long double; a (lda) is overwritten with H, alpha with diag(R), both rounded to double.  With nrhs > 0 the
 * right-hand sides b (m x nrhs, ldb) go through the long double factorisation too: qtb = Q'b (m x nrhs, leading dimension m),
 * qb = Qb (same shape) and x = H \ b (S:317-321; n x nrhs, leading dimension n).  Any of qtb, qb, x may be NULL. */
int dhqr_oracle_qr_ext(int64_t m, int64_t n, double *a, int64_t lda, double *alpha, int nrhs, const double *b, int64_t ldb,
                       double *qtb, double *qb, double *x, int nthreads) {
    if (m < 0) return -1;
    if (n < 0 || n > m) return -2;
    if (lda < (m > 1 ? m : 1)) return -4;
    if (nrhs > 0 && (!b || ldb < m)) return -5;
    if (nthreads < 1) nthreads = dhqr_oracle_max_threads();
    ldbl *w = (ldbl *)malloc(sizeof(ldbl) * (size_t)(m > 0 ? m : 1) * (size_t)(n > 0 ? n : 1));
    ldbl *al = (ldbl *)malloc(sizeof(ldbl) * (size_t)(n > 0 ? n : 1));
    ldbl *v = (ldbl *)malloc(sizeof(ldbl) * (size_t)(m > 0 ? m : 1));
    if (!w || !al || !v) { free(w); free(al); free(v); return -100; }
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < m; ++i) w[i + j * m] = a[i + j * lda];
    ext_factor(m, n, w, al, nthreads);
    for (int64_t j = 0; j < n; ++j) {
        alpha[j] = (double)al[j];
        for (int64_t i = 0; i < m; ++i) a[i + j * lda] = (double)w[i + j * m];
    }
    for (int r = 0; r < nrhs; ++r) {
        const double *br = b + (int64_t)r * ldb;
        if (qb) {
            for (int64_t i = 0; i < m; ++i) v[i] = br[i];
            ext_apply(m, n, w, v, 0);
            for (int64_t i = 0; i < m; ++i) qb[i + (int64_t)r * m] = (double)v[i];
        }
        for (int64_t i = 0; i < m; ++i) v[i] = br[i];
        ext_apply(m, n, w, v, 1);                                      /* S:288 */
        if (qtb)
            for (int64_t i = 0; i < m; ++i) qtb[i + (int64_t)r * m] = (double)v[i];
        if (x) {
            ext_backsolve(m, n, w, al, v);                             /* S:291 */
            for (int64_t i = 0; i < n; ++i) x[i + (int64_t)r * n] = (double)v[i];
        }
    }
    free(w); free(al); free(v);
    return 0;
}

/* ComplexF64 twin (S:9, S:51-59, S:162-196), real and imaginary parts kept as separate long doubles.  Interleaved complex128
 * in and out; same arguments as dhqr_oracle_qr_ext without qb (the library's apply_q_ is Float64 only). */
int dhqr_oracle_qr_ext_c(int64_t m, int64_t n, double *a, int64_t lda, double *alpha, int nrhs, const double *b, int64_t ldb,
                         double *qtb, double *x, int nthreads) {
    if (m < 0) return -1;
    if (n < 0 || n > m) return -2;
    if (lda < (m > 1 ? m : 1)) return -4;
    if (nrhs > 0 && (!b || ldb < m)) return -5;
    if (nthreads < 1) nthreads = dhqr_oracle_max_threads();
    const size_t mn = (size_t)(m > 0 ? m : 1) * (size_t)(n > 0 ? n : 1);
    ldbl *wr = (ldbl *)malloc(sizeof(ldbl) * mn), *wi = (ldbl *)malloc(sizeof(ldbl) * mn);
    ldbl *ar = (ldbl *)malloc(sizeof(ldbl) * (size_t)(n > 0 ? n : 1)), *ai = (ldbl *)malloc(sizeof(ldbl) * (size_t)(n > 0 ? n : 1));
    ldbl *vr = (ldbl *)malloc(sizeof(ldbl) * (size_t)(m > 0 ? m : 1)), *vi = (ldbl *)malloc(sizeof(ldbl) * (size_t)(m > 0 ? m : 1));
    if (!wr || !wi || !ar || !ai || !vr || !vi) { free(wr); free(wi); free(ar); free(ai); free(vr); free(vi); return -100; }
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < m; ++i) {
            wr[i + j * m] = a[2 * (i + j * lda)];
            wi[i + j * m] = a[2 * (i + j * lda) + 1];
        }
    for (int64_t j = 0; j < n; ++j) {
        ldbl *cr = wr + j * m, *ci = wi + j * m;
        ldbl s = 0.0L;
        for (int64_t i = j; i < m; ++i) s += cr[i] * cr[i] + ci[i] * ci[i];
        s = sqrtl(s);                                                  /* S:129 */
        const ldbl xr = cr[j], xi = ci[j], ax = hypotl(xr, xi);
        /* S:130, S:9: alpha = -exp(im*angle(x)) * s.  angle = atan2(im, re) sees the signs of a zero x: +-0 for +0 +- 0i,
         * +-pi for -0 +- 0i, whose (cos, sin) is (-1, +-sin(pi)) with Float64's sin(pi), as in the reference */
        const ldbl ux = ax > 0.0L ? xr / ax : (signbit(xr) ? -1.0L : 1.0L);
        const ldbl uy = ax > 0.0L ? xi / ax : (signbit(xr) ? copysignl((ldbl)1.2246467991473532e-16, xi) : xi);
        ar[j] = -s * ux;
        ai[j] = -s * uy;
        const ldbl f = 1.0L / sqrtl(s * (s + ax));                    /* S:131 */
        cr[j] -= ar[j];                                                /* S:132 */
        ci[j] -= ai[j];
        for (int64_t i = j; i < m; ++i) { cr[i] *= f; ci[i] *= f; }    /* S:133-135 */
#pragma omp parallel for schedule(static) num_threads(nthreads)
        for (int64_t jj = j + 1; jj < n; ++jj) {
            ldbl *dr = wr + jj * m, *di = wi + jj * m;
            ldbl tr = 0.0L, ti = 0.0L;                                 /* S:51-59: sum conj(v) d */
            for (int64_t i = j; i < m; ++i) {
                tr += cr[i] * dr[i] + ci[i] * di[i];
                ti += cr[i] * di[i] - ci[i] * dr[i];
            }
            for (int64_t i = j; i < m; ++i) {                          /* S:162-196: d -= v t */
                dr[i] -= cr[i] * tr - ci[i] * ti;
                di[i] -= cr[i] * ti + ci[i] * tr;
            }
        }
    }
    for (int64_t j = 0; j < n; ++j) {
        alpha[2 * j] = (double)ar[j];
        alpha[2 * j + 1] = (double)ai[j];
        for (int64_t i = 0; i < m; ++i) {
            a[2 * (i + j * lda)] = (double)wr[i + j * m];
            a[2 * (i + j * lda) + 1] = (double)wi[i + j * m];
        }
    }
    for (int r = 0; r < nrhs; ++r) {
        const double *br = b + 2 * (int64_t)r * ldb;
        for (int64_t i = 0; i < m; ++i) { vr[i] = br[2 * i]; vi[i] = br[2 * i + 1]; }
        for (int64_t j = 0; j < n; ++j) {                              /* S:232-242 with the complex partialdot */
            const ldbl *cr = wr + j * m, *ci = wi + j * m;
            ldbl tr = 0.0L, ti = 0.0L;
            for (int64_t i = j; i < m; ++i) {
                tr += cr[i] * vr[i] + ci[i] * vi[i];
                ti += cr[i] * vi[i] - ci[i] * vr[i];
            }
            for (int64_t i = j; i < m; ++i) {
                vr[i] -= cr[i] * tr - ci[i] * ti;
                vi[i] -= cr[i] * ti + ci[i] * tr;
            }
        }
        if (qtb)
            for (int64_t i = 0; i < m; ++i) { qtb[2 * (i + (int64_t)r * m)] = (double)vr[i]; qtb[2 * (i + (int64_t)r * m) + 1] = (double)vi[i]; }
        if (x) {
            for (int64_t i = n - 1; i >= 0; --i) {                     /* S:256-282, no conjugation */
                ldbl sr = 0.0L, si = 0.0L;
                for (int64_t k = i + 1; k < n; ++k) {
                    const ldbl hr = wr[i + k * m], hi = wi[i + k * m];
                    sr += hr * vr[k] - hi * vi[k];
                    si += hr * vi[k] + hi * vr[k];
                }
                const ldbl nr = vr[i] - sr, ni = vi[i] - si, d = ar[i] * ar[i] + ai[i] * ai[i];
                vr[i] = (nr * ar[i] + ni * ai[i]) / d;
                vi[i] = (ni * ar[i] - nr * ai[i]) / d;
            }
            for (int64_t i = 0; i < n; ++i) { x[2 * (i + (int64_t)r * n)] = (double)vr[i]; x[2 * (i + (int64_t)r * n) + 1] = (double)vi[i]; }
        }
    }
    free(wr); free(wi); free(ar); free(ai); free(vr); free(vi);
    return 0;
}

/* Synthetic inputs: A[i,j] ~ U[0,1) mirroring rand(T,m,n) at test/runtests.jl:45-46.  Julia's
 * stream cannot be reproduced without Julia, so entries come from a counter-based generator
 * keyed on (seed, i, j): every rank, the GPU fill kernel and numpy produce bit-identical values. */
static inline uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
double dhqr_oracle_uniform(uint64_t seed, uint64_t i, uint64_t j) {
    uint64_t z = mix64(mix64(seed) ^ (j * 0xD1342543DE82EF95ULL + i));
    return (double)(z >> 11) * 0x1.0p-53;
}
void dhqr_oracle_fill_uniform(uint64_t seed, int64_t i0, int64_t j0, int64_t m, int64_t n, double *a,
                              int64_t lda) {
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < m; ++i)
            a[i + j * lda] = dhqr_oracle_uniform(seed, (uint64_t)(i0 + i), (uint64_t)(j0 + j));
}
