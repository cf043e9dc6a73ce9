/*
 * cod_ext.c — extended-precision reference for the minimum-norm least-squares solution through the complete orthogonal
 * decomposition on a pivoted QR (test infrastructure only; compiled at test time by tests/cod_model.py into a temporary directory,
 * never linked into the product).
 *
 * It reuses the long-double column step and trailing update of adjoint_ext.c (factor(): the reference recurrences S:127-135 and
 * S:208-209, rounded to double only when written out), included here so that both references run the same recurrence.
 */
#include "adjoint_ext.c"

/* The minimum-norm solution of the rank-r least-squares problem through the complete orthogonal decomposition on a pivoted QR
 * (DESIGN §2.8), in long double with no rounding between the stages.  ap = A[:, p] (m x n, the columns in pivot order, Float64):
 * its first r reflectors (the column step and trailing update of factor() on the first r columns, then the same r reflectors on
 * columns r..n-1), c = (H_r ... H_1 b)[0:r], the factorisation of R_r' = (rows [0, r) of R)' (n x r) = Z [U; 0], z = U^{-T} c and
 * u = Z [z; 0] = H'_1 ... H'_r [z; 0].  u: n x nrhs (leading dimension n) is P'x; the permutation x[p] = u is left to the caller.
 * Returns 0, or -(argument) for a bad size, -100 when out of memory. */
int cod_ext(int64_t m, int64_t n, int64_t r, const double *ap, int64_t lda, int nrhs, const double *b, int64_t ldb, double *u,
            int nthreads) {
    if (m < 0) return -1;
    if (n < 0 || n > m) return -2;
    if (r < 0 || r > n) return -3;
    if (lda < (m > 1 ? m : 1)) return -5;
    if (nrhs > 0 && ((m > 0 && !b) || ldb < m)) return -8;
    if (nthreads < 1) nthreads = 1;
    const size_t m1 = (size_t)(m > 0 ? m : 1), n1 = (size_t)(n > 0 ? n : 1), r1 = (size_t)(r > 0 ? r : 1);
    ldbl *w = malloc(sizeof(ldbl) * m1 * n1), *al = malloc(sizeof(ldbl) * n1), *g = malloc(sizeof(ldbl) * n1 * r1);
    ldbl *ga = malloc(sizeof(ldbl) * r1), *v = malloc(sizeof(ldbl) * m1);
    if (!w || !al || !g || !ga || !v) { free(w); free(al); free(g); free(ga); free(v); return -100; }
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < m; ++i) w[i + j * m] = ap[i + j * lda];
    factor(m, r, w, NULL, al, NULL, nthreads);
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (int64_t cc = r; cc < n; ++cc) {                               /* R12: the first r reflectors on the other columns */
        ldbl *d = w + cc * m;
        for (int64_t j = 0; j < r; ++j) {
            const ldbl *h = w + j * m;
            ldbl t = 0.0L;
            for (int64_t i = j; i < m; ++i) t += h[i] * d[i];
            for (int64_t i = j; i < m; ++i) d[i] -= h[i] * t;
        }
    }
    for (int64_t i = 0; i < r; ++i)                                    /* g = R_r': g[j, i] = R[i, j] */
        for (int64_t j = 0; j < n; ++j) g[j + i * n] = j > i ? w[i + j * m] : (j == i ? al[i] : 0.0L);
    factor(n, r, g, NULL, ga, NULL, nthreads);
    for (int rr = 0; rr < nrhs; ++rr) {
        for (int64_t i = 0; i < m; ++i) v[i] = b[i + (int64_t)rr * ldb];
        for (int64_t j = 0; j < r; ++j) {                              /* c = (H_r ... H_1 b)[0:r] */
            const ldbl *h = w + j * m;
            ldbl t = 0.0L;
            for (int64_t i = j; i < m; ++i) t += h[i] * v[i];
            for (int64_t i = j; i < m; ++i) v[i] -= h[i] * t;
        }
        for (int64_t i = 0; i < r; ++i) {                              /* z = U^{-T} c, first row to last */
            ldbl s = 0.0L;
            for (int64_t j = 0; j < i; ++j) s += g[j + i * n] * v[j];
            v[i] = (v[i] - s) / ga[i];
        }
        for (int64_t i = r; i < n; ++i) v[i] = 0.0L;
        for (int64_t j = r - 1; j >= 0; --j) {                         /* u = Z [z; 0]: the reflectors of R_r' in reverse order */
            const ldbl *h = g + j * n;
            ldbl t = 0.0L;
            for (int64_t i = j; i < n; ++i) t += h[i] * v[i];
            for (int64_t i = j; i < n; ++i) v[i] -= h[i] * t;
        }
        for (int64_t i = 0; i < n; ++i) u[i + (int64_t)rr * n] = (double)v[i];
    }
    free(w); free(al); free(g); free(ga); free(v);
    return 0;
}
