/*
 * cod_ext_c.c — extended-precision reference for the ComplexF64 minimum-norm least-squares solution through the complete orthogonal
 * decomposition on a pivoted QR (test infrastructure only; compiled at test time by tests/cod_c_model.py into a temporary
 * directory, never linked into the product).  The complex twin of cod_ext.c.
 *
 * It reuses the long-double complex column step and trailing update of adjoint_ext.c (factor() with separate real and imaginary
 * parts, rounded to double only when written out), included here so that every reference runs the same recurrence.
 */
#include "adjoint_ext.c"

/* (vr + i vi)[j:len] -= h (h^H v)[j:len] for the reflector h = (hr + i hi), rows j..len-1 */
static void reflect_c(int64_t j, int64_t len, const ldbl *hr, const ldbl *hi, ldbl *vr, ldbl *vi) {
    ldbl tr = 0.0L, ti = 0.0L;
    for (int64_t i = j; i < len; ++i) {
        tr += hr[i] * vr[i] + hi[i] * vi[i];
        ti += hr[i] * vi[i] - hi[i] * vr[i];
    }
    for (int64_t i = j; i < len; ++i) {
        vr[i] -= hr[i] * tr - hi[i] * ti;
        vi[i] -= hr[i] * ti + hi[i] * tr;
    }
}

/* x = P Z [U^{-H} (Q^H b)[0:r]; 0] in long double, ComplexF64 in and out (interleaved).  ap = A[:, p] (m x n, lda), b (m x nrhs,
 * ldb); the stages as in cod_ext with conjugate transposes: G = R_r^H (n x r, G[j, i] = conj(R[i, j])) = Z [U; 0], z = U^{-H} c with
 * z_i = (c_i - sum_{j<i} conj(U[j, i]) z_j) / conj(U[i, i]), u = Z [z; 0].  u: n x nrhs (leading dimension n) is P'x.  Returns 0,
 * or -(argument) for a bad size, -100 when out of memory. */
int cod_ext_c(int64_t m, int64_t n, int64_t r, const double *ap, int64_t lda, int nrhs, const double *b, int64_t ldb, double *u,
              int nthreads) {
    if (m < 0) return -1;
    if (n < 0 || n > m) return -2;
    if (r < 0 || r > n) return -3;
    if (lda < (m > 1 ? m : 1)) return -5;
    if (nrhs > 0 && ((m > 0 && !b) || ldb < m)) return -8;
    if (nthreads < 1) nthreads = 1;
    const size_t m1 = (size_t)(m > 0 ? m : 1), n1 = (size_t)(n > 0 ? n : 1), r1 = (size_t)(r > 0 ? r : 1);
    ldbl *wr = malloc(sizeof(ldbl) * m1 * n1), *wi = malloc(sizeof(ldbl) * m1 * n1);
    ldbl *alr = malloc(sizeof(ldbl) * n1), *ali = malloc(sizeof(ldbl) * n1);
    ldbl *gr = malloc(sizeof(ldbl) * n1 * r1), *gi = malloc(sizeof(ldbl) * n1 * r1);
    ldbl *gar = malloc(sizeof(ldbl) * r1), *gai = malloc(sizeof(ldbl) * r1);
    ldbl *vr = malloc(sizeof(ldbl) * m1), *vi = malloc(sizeof(ldbl) * m1);
    if (!wr || !wi || !alr || !ali || !gr || !gi || !gar || !gai || !vr || !vi) {
        free(wr); free(wi); free(alr); free(ali); free(gr); free(gi); free(gar); free(gai); free(vr); free(vi);
        return -100;
    }
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < m; ++i) {
            wr[i + j * m] = ap[2 * (i + j * lda)];
            wi[i + j * m] = ap[2 * (i + j * lda) + 1];
        }
    factor(m, r, wr, wi, alr, ali, nthreads);
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (int64_t cc = r; cc < n; ++cc)                                 /* R12: the first r reflectors on the other columns */
        for (int64_t j = 0; j < r; ++j) reflect_c(j, m, wr + j * m, wi + j * m, wr + cc * m, wi + cc * m);
    for (int64_t i = 0; i < r; ++i)                                    /* G = R_r^H: G[j, i] = conj(R[i, j]) */
        for (int64_t j = 0; j < n; ++j) {
            gr[j + i * n] = j > i ? wr[i + j * m] : (j == i ? alr[i] : 0.0L);
            gi[j + i * n] = j > i ? -wi[i + j * m] : (j == i ? -ali[i] : 0.0L);
        }
    factor(n, r, gr, gi, gar, gai, nthreads);
    for (int rr = 0; rr < nrhs; ++rr) {
        for (int64_t i = 0; i < m; ++i) {
            vr[i] = b[2 * (i + (int64_t)rr * ldb)];
            vi[i] = b[2 * (i + (int64_t)rr * ldb) + 1];
        }
        for (int64_t j = 0; j < r; ++j) reflect_c(j, m, wr + j * m, wi + j * m, vr, vi);    /* c = (H_r ... H_1 b)[0:r] */
        for (int64_t i = 0; i < r; ++i) {                              /* z = U^{-H} c, first row to last */
            ldbl sr = 0.0L, si = 0.0L;
            for (int64_t j = 0; j < i; ++j) {                          /* conj(U[j, i]) z_j */
                const ldbl ur = gr[j + i * n], ui = -gi[j + i * n];
                sr += ur * vr[j] - ui * vi[j];
                si += ur * vi[j] + ui * vr[j];
            }
            const ldbl nr = vr[i] - sr, ni = vi[i] - si, dr = gar[i], di = -gai[i], d = dr * dr + di * di;
            vr[i] = (nr * dr + ni * di) / d;
            vi[i] = (ni * dr - nr * di) / d;
        }
        for (int64_t i = r; i < n; ++i) vr[i] = vi[i] = 0.0L;
        for (int64_t j = r - 1; j >= 0; --j) reflect_c(j, n, gr + j * n, gi + j * n, vr, vi);   /* u = Z [z; 0] */
        for (int64_t i = 0; i < n; ++i) {
            u[2 * (i + (int64_t)rr * n)] = (double)vr[i];
            u[2 * (i + (int64_t)rr * n) + 1] = (double)vi[i];
        }
    }
    free(wr); free(wi); free(alr); free(ali); free(gr); free(gi); free(gar); free(gai); free(vr); free(vi);
    return 0;
}
