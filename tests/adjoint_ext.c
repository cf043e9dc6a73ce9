/*
 * adjoint_ext.c — extended-precision reference for the solves with the adjoint (test infrastructure only; compiled at test
 * time by tests/adjoint_oracle.py into a temporary directory, never linked into the product).
 *
 * The reference recurrences in long double, rounded to double only when written out, as in oracle/dhqr_oracle.c's qr_ext:
 * the column step S:127-135 (alphafactor S:8 / S:9), the trailing update S:208-209 with the conjugating partialdot S:51-59,
 * then for every right-hand side c
 *     z = R^{-H} c           z_i = (c_i - sum_{j<i} conj(R[j,i]) z_j) / conj(alpha_i)
 *     y = Q [z; 0]           Q = H_1 ... H_n: the reflectors in reverse order
 * y is the minimum-norm solution of A^H y = c.  Each trailing column is updated by one thread with a sequential sum, so the
 * result does not depend on the thread count.  Real and imaginary parts are separate long doubles; wi == NULL is Float64.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef long double ldbl;

static void factor(int64_t m, int64_t n, ldbl *wr, ldbl *wi, ldbl *ar, ldbl *ai, int nthreads) {
    for (int64_t j = 0; j < n; ++j) {
        ldbl *cr = wr + j * m, *ci = wi ? wi + j * m : NULL;
        ldbl s = 0.0L;
        for (int64_t i = j; i < m; ++i) s += cr[i] * cr[i] + (ci ? ci[i] * ci[i] : 0.0L);
        s = sqrtl(s);                                                   /* S:129 */
        const ldbl xr = cr[j], xi = ci ? ci[j] : 0.0L, ax = ci ? hypotl(xr, xi) : fabsl(xr);
        if (ci) {                                                       /* S:9: -exp(i angle(x)) s, angle(-0 +- 0i) = +-pi */
            ar[j] = -s * (ax > 0.0L ? xr / ax : (signbit(xr) ? -1.0L : 1.0L));
            ai[j] = -s * (ax > 0.0L ? xi / ax : (signbit(xr) ? copysignl((ldbl)1.2246467991473532e-16, xi) : xi));
        } else {                                                        /* S:8: -sign(x) s, sign(0) = 0 */
            ar[j] = s * (xr > 0.0L ? -1.0L : (xr < 0.0L ? 1.0L : -0.0L * 0.0L));
        }
        const ldbl f = 1.0L / sqrtl(s * (s + ax));                     /* S:131 */
        cr[j] -= ar[j];                                                 /* S:132 */
        if (ci) ci[j] -= ai[j];
        for (int64_t i = j; i < m; ++i) {                               /* S:133-135 */
            cr[i] *= f;
            if (ci) ci[i] *= f;
        }
#pragma omp parallel for schedule(static) num_threads(nthreads)
        for (int64_t jj = j + 1; jj < n; ++jj) {
            ldbl *dr = wr + jj * m, *di = wi ? wi + jj * m : NULL;
            ldbl tr = 0.0L, ti = 0.0L;                                  /* S:51-59: sum conj(v) d */
            for (int64_t i = j; i < m; ++i) {
                tr += cr[i] * dr[i] + (ci ? ci[i] * di[i] : 0.0L);
                if (ci) ti += cr[i] * di[i] - ci[i] * dr[i];
            }
            for (int64_t i = j; i < m; ++i) {                           /* S:162-196 / S:209: d -= v t */
                dr[i] -= cr[i] * tr - (ci ? ci[i] * ti : 0.0L);
                if (ci) di[i] -= cr[i] * ti + ci[i] * tr;
            }
        }
    }
}

/* a: m x n (lda), complex interleaved when cplx; c: n x nrhs (ldc >= n); z: n x nrhs (leading dimension n) and y: m x nrhs
 * (leading dimension m), either may be NULL.  Returns 0, or -(argument) for a bad size, -100 when out of memory. */
int adj_ext(int64_t m, int64_t n, const double *a, int64_t lda, int cplx, int nrhs, const double *c, int64_t ldc, double *z,
            double *y, int nthreads) {
    if (m < 0) return -1;
    if (n < 0 || n > m) return -2;
    if (lda < (m > 1 ? m : 1)) return -4;
    if (nrhs > 0 && ((n > 0 && !c) || ldc < n)) return -7;
    if (nthreads < 1) nthreads = 1;
    const int e = cplx ? 2 : 1;
    const size_t mn = (size_t)(m > 0 ? m : 1) * (size_t)(n > 0 ? n : 1), n1 = (size_t)(n > 0 ? n : 1), m1 = (size_t)(m > 0 ? m : 1);
    ldbl *wr = malloc(sizeof(ldbl) * mn), *wi = cplx ? malloc(sizeof(ldbl) * mn) : NULL;
    ldbl *ar = malloc(sizeof(ldbl) * n1), *ai = malloc(sizeof(ldbl) * n1);
    ldbl *vr = malloc(sizeof(ldbl) * m1), *vi = malloc(sizeof(ldbl) * m1);
    if (!wr || (cplx && !wi) || !ar || !ai || !vr || !vi) { free(wr); free(wi); free(ar); free(ai); free(vr); free(vi); return -100; }
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < m; ++i) {
            wr[i + j * m] = a[e * (i + j * lda)];
            if (cplx) wi[i + j * m] = a[e * (i + j * lda) + 1];
        }
    for (int64_t j = 0; j < n; ++j) ai[j] = 0.0L;
    factor(m, n, wr, wi, ar, cplx ? ai : NULL, nthreads);
    for (int r = 0; r < nrhs; ++r) {
        const double *cc = c + (int64_t)e * r * ldc;
        for (int64_t i = 0; i < n; ++i) {                               /* z = R^{-H} c, first row to last */
            ldbl sr = 0.0L, si = 0.0L;
            for (int64_t j = 0; j < i; ++j) {
                const ldbl hr = wr[j + i * m], hi = cplx ? wi[j + i * m] : 0.0L;
                sr += hr * vr[j] + hi * vi[j];
                si += hr * vi[j] - hi * vr[j];
            }
            const ldbl nr = cc[e * i] - sr, ni = (cplx ? cc[e * i + 1] : 0.0L) - si, d = ar[i] * ar[i] + ai[i] * ai[i];
            vr[i] = (nr * ar[i] - ni * ai[i]) / d;                      /* (nr + i ni) / conj(alpha) */
            vi[i] = (ni * ar[i] + nr * ai[i]) / d;
        }
        if (z)
            for (int64_t i = 0; i < n; ++i) {
                z[e * (i + (int64_t)r * n)] = (double)vr[i];
                if (cplx) z[e * (i + (int64_t)r * n) + 1] = (double)vi[i];
            }
        for (int64_t i = n; i < m; ++i) vr[i] = vi[i] = 0.0L;
        for (int64_t j = n - 1; j >= 0; --j) {                          /* y = H_1 ... H_n [z; 0] */
            const ldbl *hr = wr + j * m, *hi = cplx ? wi + j * m : NULL;
            ldbl tr = 0.0L, ti = 0.0L;
            for (int64_t i = j; i < m; ++i) {
                tr += hr[i] * vr[i] + (hi ? hi[i] * vi[i] : 0.0L);
                ti += hr[i] * vi[i] - (hi ? hi[i] * vr[i] : 0.0L);
            }
            for (int64_t i = j; i < m; ++i) {
                vr[i] -= hr[i] * tr - (hi ? hi[i] * ti : 0.0L);
                vi[i] -= hr[i] * ti + (hi ? hi[i] * tr : 0.0L);
            }
        }
        if (y)
            for (int64_t i = 0; i < m; ++i) {
                y[e * (i + (int64_t)r * m)] = (double)vr[i];
                if (cplx) y[e * (i + (int64_t)r * m) + 1] = (double)vi[i];
            }
    }
    free(wr); free(wi); free(ar); free(ai); free(vr); free(vi);
    return 0;
}
