/*
 * downdate_ext.c — extended-precision reference for the downdate (test infrastructure only; compiled at test time by
 * tests/downdate_model.py into a temporary directory, never linked into the product).
 *
 * The unblocked hyperbolic recurrence of DESIGN §2.11 in long double, rounded to double only when written out.  Column j of
 * [R; Z] with x0 = R[j, j] (alpha[j]) and t = ||Z[:, j]||^2:
 *     sigma^2 = (|x0| - sqrt(t)) (|x0| + sqrt(t)),  alpha = -sign(x0) sigma (zero x0 positive),  f = 1 / sqrt(sigma (sigma + |x0|)),
 *     vtop = f (x0 - alpha),  V2 = f Z[:, j],  w_c = vtop R[j, c] - V2' Z[:, c],  R[j, c] -= vtop w_c,  Z[:, c] -= V2 w_c,
 * and the same w / update on the right-hand sides [c; e].  The first column with sigma^2 <= 0 while t > 0, or a NaN sigma^2, is
 * returned (1-based); it and every later column store vtop = 0, V2 = 0, alpha = NaN and change nothing.  A zero column (sigma = 0,
 * t = 0) stores zeros.  All arrays are column-major with leading dimension n (R, c) or k (Z, e); everything is overwritten in place.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef long double ldbl;

int64_t downdate_ext(int64_t n, int64_t k, double *R, double *alpha, double *Z, double *vtop, double *c, double *e, int64_t nrhs) {
    ldbl *r = malloc(sizeof(ldbl) * (size_t)(n * n + 1)), *z = malloc(sizeof(ldbl) * (size_t)(k * n + 1));
    ldbl *cc = malloc(sizeof(ldbl) * (size_t)(n * nrhs + 1)), *ee = malloc(sizeof(ldbl) * (size_t)(k * nrhs + 1));
    for (int64_t i = 0; i < n * n; ++i) r[i] = R[i];
    for (int64_t i = 0; i < n; ++i) r[i * n + i] = alpha[i];
    for (int64_t i = 0; i < k * n; ++i) z[i] = Z[i];
    for (int64_t i = 0; i < n * nrhs; ++i) cc[i] = c[i];
    for (int64_t i = 0; i < k * nrhs; ++i) ee[i] = e[i];
    int64_t info = 0;
    for (int64_t j = 0; j < n; ++j) {
        ldbl *zj = z + j * k, t = 0.0L;
        for (int64_t i = 0; i < k; ++i) t += zj[i] * zj[i];
        const ldbl x0 = r[j * n + j], ax = fabsl(x0), rt = sqrtl(t), s2 = (ax - rt) * (ax + rt);
        if (info || isnan(s2) || (t > 0.0L && s2 <= 0.0L)) {
            if (!info) info = j + 1;
            for (int64_t i = 0; i < k; ++i) zj[i] = 0.0L;
            r[j * n + j] = NAN;
            vtop[j] = 0.0;
            continue;
        }
        const ldbl s = sqrtl(s2);
        const ldbl al = s == 0.0L ? 0.0L : (x0 >= 0.0L ? -s : s);
        const ldbl f = s == 0.0L ? 0.0L : 1.0L / sqrtl(s * (s + ax));
        const ldbl vt = f * (x0 - al);
        for (int64_t i = 0; i < k; ++i) zj[i] *= f;
        for (int64_t q = j + 1; q < n + nrhs; ++q) {                   /* columns of R, then the right-hand sides */
            const int rhs = q >= n;
            ldbl *col = rhs ? ee + (q - n) * k : z + q * k, top = rhs ? cc[(q - n) * n + j] : r[q * n + j];
            ldbl d = 0.0L;
            for (int64_t i = 0; i < k; ++i) d += zj[i] * col[i];
            const ldbl w = vt * top - d;
            if (rhs) cc[(q - n) * n + j] -= vt * w; else r[q * n + j] -= vt * w;
            for (int64_t i = 0; i < k; ++i) col[i] -= zj[i] * w;
        }
        r[j * n + j] = al;
        vtop[j] = (double)vt;
    }
    for (int64_t j = 0; j < n; ++j)
        for (int64_t i = 0; i < j; ++i) R[j * n + i] = (double)r[j * n + i];
    for (int64_t i = 0; i < n; ++i) alpha[i] = (double)r[i * n + i];
    for (int64_t i = 0; i < k * n; ++i) Z[i] = (double)z[i];
    for (int64_t i = 0; i < n * nrhs; ++i) c[i] = (double)cc[i];
    for (int64_t i = 0; i < k * nrhs; ++i) e[i] = (double)ee[i];
    free(r); free(z); free(cc); free(ee);
    return info;
}
