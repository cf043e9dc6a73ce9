/*
 * dhqr.h — C-ABI of libdhqr.so: H100-native (sm_90a) blocked Householder QR behind
 * DistributedHouseholderQR.jl's qr! / \ entry points.
 *
 * The reference (pure Julia) has no FFI of its own; each entry point below names the Julia
 * method it replaces (S:n = src/DistributedHouseholderQR.jl:n of the reference).  A Julia shim
 * (distributedhouseholderqr.jl_b200/julia/DistributedHouseholderQRB200.jl, see INTEGRATION.md)
 * ccall's these with CuPtr{Float64}; the Python host package binds them with ctypes.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / CUDA.jl types in any signature.
 *   - every function returns int: 0 = ok; < 0 = -(1-based index of the offending argument),
 *     LAPACK-info style; > 0 = CUDA/NCCL failure (text via dhqr_last_error()).
 *   - matrices are column-major double with leading dimension lda >= m (Julia Matrix /
 *     localpart(DArray)).  Device pointers unless the name says _host_.
 *   - storage: any leading dimension >= max(1, m) and any base address with the element type's natural alignment: 8 B for
 *     Float64, 16 B for ComplexF64 (the _c64 entry points return -(index) for a ComplexF64 pointer that is only 8 B aligned,
 *     before anything is enqueued).  Results are bitwise independent of both.  Nothing outside the m x n operand (vector,
 *     alpha) is written, and padding rows or neighbouring data never enter a result, even when they are Inf or NaN.
 *   - stream-ordered: work is enqueued on the caller's cudaStream_t (passed as void*; NULL =
 *     legacy default stream).  Synchronisation points, all of them: (i) the _host_ entry points block
 *     until their result is in host memory; (ii) dhqr_qr_f64 with the default blocked path synchronises
 *     the stream ONCE before returning whenever a panel went through the speculative 128-column chain
 *     (option "wide_panel", on by default: its conditioning guards are evaluated on the device and a
 *     refused panel is redone by the 32-column chain); (iii) with nranks > 1 every qr / apply_qt /
 *     backsolve call exchanges the column partition first (one small all-gather + stream sync);
 *     (iv) workspace growth (first call, or a larger problem than any before) allocates device memory.
 *     Everything else returns without synchronising.  Any caller stream works, non-blocking and prioritised ones
 *     included: the library depends on no stream but the caller's (workspace zero fills included; its internal streams
 *     fork from and join back to the caller's stream with events).  tests/test_gpu_streams.py and tests/test_gpu_adjoint.py
 *     (the adjoint solves) hold every entry point to this.
 *   - no pointer to caller memory is retained after return; workspace lives in the handle.
 *   - a handle is not thread-safe and its calls share one workspace: one handle per host thread, and
 *     consecutive calls on one handle must be on the same stream or ordered by the caller (events);
 *     the library does not order calls that arrive on different streams (the reference is not
 *     re-entrant either: Polyester @batch, S:203-206).
 *   - SPMD for multi-GPU: every rank (one process per GPU) makes the same call with its own
 *     column block (col0 = first global column, 0-based = the reference's LocalColumnBlock.dj, S:34).
 *   - storage format on return == the reference's (S:127-135): Householder vectors scaled to
 *     |v|^2 = 2 in the lower trapezoid INCLUDING the diagonal, R's strict upper triangle above
 *     it, diag(R) in alpha.
 */
#ifndef DHQR_H
#define DHQR_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dhqr_context *dhqr_handle;

#define DHQR_VERSION 100 /* 0.1.0 */
#define DHQR_NCCL_UNIQUE_ID_BYTES 128

/* ---- library / handle -------------------------------------------------------------------- */
int dhqr_version(void);
/* Text of the last error raised on the calling thread ("" if none). */
const char *dhqr_last_error(void);

/* Single-GPU handle on CUDA device `device` (replaces nothing in the reference: the Julia
 * package keeps no state; the handle owns workspace and the grid-barrier words). */
int dhqr_create(dhqr_handle *h, int device);
/* Multi-GPU handle: rank `rank` of `nranks`, NCCL communicator built from `unique_id`
 * (DHQR_NCCL_UNIQUE_ID_BYTES bytes from dhqr_nccl_unique_id() on rank 0, shipped by the host:
 * torch.distributed in Python, Distributed.jl in Julia).  Replaces the reference's use of
 * Distributed/SharedArrays (S:116-118, S:141-143, S:227-229, S:260-267, S:302, S:318). */
int dhqr_create_dist(dhqr_handle *h, int device, const void *unique_id, int rank, int nranks);
int dhqr_nccl_unique_id(void *out_unique_id);
int dhqr_destroy(dhqr_handle h);
/* Tunables (dhqr_set_option / dhqr_get_option):
 *   "nb"          outer panel width, multiple of 32 in [32,128] (default 128)
 *   "lookahead"   1 (default): panel chain on a high-priority stream ahead of the bulk update; 0: one stream, serial
 *   "wide_panel"  1 (default): full, 32-aligned outer panels of width 128 are factored by the 128-column chain
 *                 (CholeskyQR2 + Householder reconstruction on the whole panel: 3 grid-wide reductions per 128 columns,
 *                 no cooperative launch); refused panels and all other panels use the 32-column chain below
 *   "panel_fast"  1 (default): inner panels by CholeskyQR2 + Householder reconstruction with on-device fallback
 *                 to the column-by-column kernel; 0: always column by column
 *   "panel_ctas"  CTAs of the cooperative panel kernel (0 = default: 64 under look-ahead, one per SM otherwise)
 *   "cvy_persist" consecutive tiles per CTA of the 128-wide trailing update (default 4; 0: one tile per CTA, same result)
 *   "qt_vec"      1 (default): Q'b / Qb with ONE right-hand side as a GEMV sweep (T' of every panel computed first, then two
 *                 HBM-bound launches per panel that read the reflectors in place); 0: the GEMM-shaped block update, as for nrhs > 1
 *   "host_chunk"  columns per upload chunk of dhqr_qr_host_f64 (default 512, a multiple of 128; 0: one upload, no overlap);
 *                 "host_h2d_gbs" (50), "host_tflops" (27), "host_chain_us" (300): what its join-step planner assumes about the
 *                 host link, the device and a step of the schedule on a narrow window; "host_cu_streams" (3): catch-up streams; "host_first" (0 = three panels): columns of the first, exposed upload;
 *                 "host_trace" 1: stage timeline on stderr.  A wrong assumption costs idle time, never correctness
 *   "sync"        1: cudaStreamSynchronize + error check after every kernel launch (debugging; implies serial)
 *   "profile"     1: CUDA-event bracket per launch (implies serial), read with dhqr_profile_get
 *   "bs_wave", "unblocked_wave", "fuse_house"  1 (default): back-substitution (and the Float64 forward substitution of
 *                 dhqr_forwardsolve_f64 / dhqr_solve_adj_f64) as one wavefront launch per right-hand side where all its CTAs fit
 *                 on the device, nb = 1 as one persistent launch (m <= 8192), nb = 1 with the next reflector formed inside the
 *                 apply kernel, where the shape allows; 0: the per-block / per-column launches those paths otherwise take
 *   "wide_kappa"  guard of the 128-column chain on ||D R1^{-1}||_F of its first Cholesky factor (default 1000)
 *   traces:       "panel_trace", "la_trace", "wide_trace" (timestamps read with dhqr_debug_copy_f64)
 *   read-only:    "sms", "rank", "nranks", "panels_fast", "panels_fallback" (inner panels taken by either path; device-side
 *                 counters of work the device has finished: read them after synchronising the stream of the calls),
 *                 "wide_panels" (outer panels factored by the 128-column chain), "wide_redone" (restarts after a refusal),
 *                 "qrcp_renorms" (exact column renorms of dhqr_qrcp_f64; device-side, read after synchronising)
 *   dhqr_get_option reads "nb", "panel_ctas", "sync", "profile", "lookahead", "panel_fast", "wide_panel", "cvy_persist",
 *                 "qt_vec", "bs_wave", "unblocked_wave", "fuse_house", "host_chunk" and the read-only keys.
 *   Any other key returns -2 (unknown option). */
int dhqr_set_option(dhqr_handle h, const char *key, int64_t value);
int dhqr_get_option(dhqr_handle h, const char *key, int64_t *value);
/* Number of kernel launches enqueued by this handle since creation (bench.py: gpu_launches). */
int dhqr_launch_count(dhqr_handle h, int64_t *count);
/* Per-kernel-class timing with CUDA events on the launching stream (option "profile" = 1 turns the
 * brackets on; the reference keeps the same kind of accumulators as t1a/t1b/t2, S:126-146, S:291).
 * dhqr_profile_get returns slot `index` (0.. until -2): class name, accumulated milliseconds, launch
 * count and algorithmic work (flops for the GEMM classes, bytes for the panel).  Blocks on the events. */
int dhqr_profile_reset(dhqr_handle h);
int dhqr_profile_get(dhqr_handle h, int index, char *name, int name_len, double *ms, int64_t *count,
                     double *work);

/* ---- qr!  (S:311-315 -> householder! S:113-120 -> _householder! S:122-148 -> _householder_inner!
 *            S:198-213 with partialdot S:42-49 and hotloop! S:156-160) --------------------------
 * Factor the m x n_global matrix whose columns [col0, col0+n_local) are stored in dA_local
 * (m x n_local, lda).  In place.  d_alpha (length n_global) receives diag(R) on every rank.
 * nb: 0 = handle default (blocked, compact-WY trailing update on the fp64 tensor pipe);
 *     1 = unblocked column-by-column path (BASELINE config 2);
 *     otherwise a multiple of 32 in [32,128]. */
int dhqr_qr_f64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                double *dA_local, int64_t lda, double *d_alpha, int nb, void *stream);

/* ---- \  (S:317-321 -> solve_householder! S:284-294) ---------------------------------------- */
/* b <- Q'b  (_solve_householder1! S:226-242 / S:215-224).  d_b: m x nrhs, ldb >= m, in place;
 * identical on every rank on entry and on return. */
int dhqr_apply_qt_f64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                      const double *dA_local, int64_t lda, double *d_b, int64_t ldb, int nrhs,
                      void *stream);
/* b <- Q b = H_1 ... H_n b: the inverse of the sweep above (not in the reference, which never forms Q; SURVEY 8f-3:
 * exposes the factorisation as an operator, e.g. to form Q explicitly or to compute residuals b - A x = Q [0; (Q'b)[n:]]). */
int dhqr_apply_q_f64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                     const double *dA_local, int64_t lda, double *d_b, int64_t ldb, int nrhs, void *stream);
/* b[0:n] <- R^{-1} b[0:n]  (_solve_householder2! S:256-282 / S:244-254), R = triu(A,1)+diag(alpha). */
int dhqr_backsolve_f64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                       const double *dA_local, int64_t lda, const double *d_alpha, double *d_b,
                       int64_t ldb, int nrhs, void *stream);
/* Both phases (solve_householder! S:284-294): x = d_b[0:n_global, :] on return. */
int dhqr_solve_f64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                   const double *dA_local, int64_t lda, const double *d_alpha, double *d_b,
                   int64_t ldb, int nrhs, void *stream);

/* ---- ComplexF64 (the reference's second element type: test/runtests.jl:43; alphafactor(::Complex) S:9, the conjugating
 * partialdot S:51-59, the complex hotloop! S:162-196).  Matrices and vectors are interleaved (re, im) doubles = Julia
 * ComplexF64 / C double _Complex; lda, ldb count COMPLEX elements; alpha is complex (length n).  Same storage format:
 * v scaled to |v|^2 = 2 in the lower trapezoid including the diagonal, H_j = I - v_j v_j^H, diag(R) in alpha.
 * Single GPU: col0 must be 0 and n_local == n_global.  Stream-ordered, no synchronisation.  Every ComplexF64 pointer (dA_local,
 * d_alpha, d_b, dQ, d_a, d_out) must be 16 B aligned: the kernels move whole (re, im) pairs; an 8 B aligned one returns minus its
 * argument index (dhqr_qr_c64: -6 / -8; apply_qt: -6 / -8; backsolve and solve: -6 / -8 / -9 for A / alpha / b; form_q_c64: -4 / -6;
 * partialdot_c64: -2 / -3 / -6) and nothing is enqueued. */
int dhqr_qr_c64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, void *dA_local,
                int64_t lda, void *d_alpha, void *stream);
int dhqr_apply_qt_c64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                      const void *dA_local, int64_t lda, void *d_b, int64_t ldb, int nrhs, void *stream);
int dhqr_backsolve_c64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                       const void *dA_local, int64_t lda, const void *d_alpha, void *d_b, int64_t ldb,
                       int nrhs, void *stream);
int dhqr_solve_c64(dhqr_handle h, int64_t m, int64_t n_global, int64_t col0, int64_t n_local,
                   const void *dA_local, int64_t lda, const void *d_alpha, void *d_b, int64_t ldb, int nrhs,
                   void *stream);
/* partialdot(a, b, is, ::Type{<:Complex}) (S:51-59): *d_out = sum_{i in [i0,i1)} conj(a[i]) * b[i]. */
int dhqr_partialdot_c64(dhqr_handle h, const void *d_a, const void *d_b, int64_t i0, int64_t i1, void *d_out,
                        void *stream);

/* ---- explicit thin Q (not in the reference, which never forms Q; SURVEY 8f-3, the second half of Q as an operator) ----------
 * Q <- the first n columns of Q = H_1 H_2 ... H_n, i.e. Q [I_n; 0] (LAPACK orgqr / ungqr), from a factorisation (dA, lda) in
 * the library's storage format (any path: blocked, nb = 1, ComplexF64).  dQ: m x n, ldq >= m; written, never read on entry.
 * dQ == dA with ldq == lda overwrites the factorisation with Q (R is lost: read it first); any other overlap of the two is
 * rejected.  Whatever reflectors are stored are used as they are: after an exact zero pivot of nb = 1 (INTEGRATION.md) that is
 * H_1 ... H_n [I; 0] of those reflectors.  Single GPU (a handle with nranks > 1 returns -1).  Stream-ordered, no synchronisation
 * apart from workspace growth (point (iv)).  Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 / -6 null
 * matrix with n > 0, -5 / -7 leading dimension < max(1, m), -6 dQ overlaps dA without being it, or dQ == dA with ldq != lda.
 * n = 0 is a no-op. */
int dhqr_form_q_f64(dhqr_handle h, int64_t m, int64_t n, const double *dA, int64_t lda, double *dQ, int64_t ldq,
                    void *stream);
/* ComplexF64: interleaved (re, im); lda, ldq in complex elements.  Q = H_1 ... H_n with H_j = I - v_j v_j^H. */
int dhqr_form_q_c64(dhqr_handle h, int64_t m, int64_t n, const void *dA, int64_t lda, void *dQ, int64_t ldq,
                    void *stream);

/* ---- solves with the adjoint (not in the reference; SURVEY 8f-3: LAPACK ?gels with TRANS = 'C', full rank) -------------------
 * From a factorisation A = QR (dA, lda, d_alpha) in the library's storage format, R = triu(A, 1) + diag(alpha), any path.
 * d_b: m x nrhs, ldb >= max(1, m), in place.  Single GPU (a handle with nranks > 1 returns -1).  Stream-ordered, no
 * synchronisation apart from workspace growth (point (iv)).  Nothing outside the m x nrhs operand b is written; A and alpha
 * never are.  A zero entry of alpha divides by zero and propagates Inf / NaN, as in dhqr_backsolve_*.
 * Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 null A with n > 0, -5 lda < max(1, m), -6 null alpha
 * with n > 0, -7 null b with nrhs > 0, -8 ldb < max(1, m), -9 nrhs < 0; the _c64 functions also return -4 / -6 / -7 for an A,
 * alpha or b that is only 8 B aligned.  Every check runs before anything is enqueued.
 *
 * b[0:n, :] <- R^{-H} b[0:n, :] (R^{-T} for Float64): forward substitution with the lower-triangular R^H.  Rows n..m-1 of b are
 * neither read nor written.  n = 0 is a no-op. */
int dhqr_forwardsolve_f64(dhqr_handle h, int64_t m, int64_t n, const double *dA, int64_t lda, const double *d_alpha,
                          double *d_b, int64_t ldb, int nrhs, void *stream);
int dhqr_forwardsolve_c64(dhqr_handle h, int64_t m, int64_t n, const void *dA, int64_t lda, const void *d_alpha, void *d_b,
                          int64_t ldb, int nrhs, void *stream);
/* Minimum-norm solution of A^H y = c: on entry c = b[0:n, :]; on return y = b[0:m, :] = Q [R^{-H} c; 0].  n = 0 sets the
 * m x nrhs block of b to zero (the minimum-norm solution of an empty system, as in ?gels). */
int dhqr_solve_adj_f64(dhqr_handle h, int64_t m, int64_t n, const double *dA, int64_t lda, const double *d_alpha, double *d_b,
                       int64_t ldb, int nrhs, void *stream);
int dhqr_solve_adj_c64(dhqr_handle h, int64_t m, int64_t n, const void *dA, int64_t lda, const void *d_alpha, void *d_b,
                       int64_t ldb, int nrhs, void *stream);

/* ---- QR with column pivoting (not in the reference; LAPACK dgeqp3 + dgelsy's basic solution) ---------------------------------
 * A P = Q R: Householder QR with Businger-Golub pivoting on the largest remaining column norm, blocked as in LAPACK dlaqps
 * (panels of 32 columns, partial norms downdated with LAPACK's tol3z = sqrt(eps) test; a column that fails it is renormed exactly
 * before the next pivot is chosen).  Float64, single GPU (a handle with nranks > 1 returns -1), n <= m, no row limit.
 * Stream-ordered, no synchronisation apart from workspace growth (point (iv)).  Two calls on the same input give bitwise
 * identical results.  Nothing outside A (m x n), alpha (n) or jpvt (n) is written, and no pointer may be less than 8 B aligned.
 *
 * dhqr_qrcp_f64: factors in place.  On return A[:, jpvt] = Q R in the library's storage format, so (dA, lda, d_alpha) is the
 * factorisation of the permuted matrix for every other entry point (apply_qt / apply_q / backsolve / form_q / forwardsolve);
 * jpvt is 0-based: jpvt[k] = original index of the k-th column.  Pivot k is the remaining column with the largest partial norm;
 * a tie goes to the smallest index, a NaN norm beats every number (so NaN input shows up in alpha[0]).  alpha_k = -sign(x0) ||x||
 * with a zero x0 counted as positive.  Once the largest remaining norm is exactly 0, every remaining column is zero in working
 * precision and every remaining step stores v = 0 and alpha = 0 (H = I).  Read-only option "qrcp_renorms": exact renorms so far.
 * Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 null (n > 0) or misaligned A, -5 lda < max(1, m),
 * -6 null or misaligned alpha, -7 null or misaligned jpvt.  Every check runs before anything is enqueued.  n = 0 is a no-op. */
int dhqr_qrcp_f64(dhqr_handle h, int64_t m, int64_t n, double *dA, int64_t lda, double *d_alpha, int64_t *d_jpvt, void *stream);
/* x = P [R11^{-1} (Q'b)[0:rank]; 0]: the basic solution of min ||A x - b|| at the given rank (LAPACK dgelsy without the complete
 * orthogonal decomposition), from a factorisation made by dhqr_qrcp_f64.  Choosing the rank needs alpha on the host, so it is an
 * argument.  d_b: m x nrhs, ldb >= max(1, m), in place: on return b[0:n] = x, and rows n..m-1 hold rows n..m-1 of
 * H_rank ... H_1 b.  Only the first `rank` reflectors run.  rank = 0 gives x = 0.  jpvt entries outside [0, n) are skipped, so
 * nothing is ever written outside b.  Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 rank < 0 or
 * rank > n, -5 null or misaligned A, -6 lda < max(1, m), -7 null or misaligned alpha, -8 null or misaligned jpvt, -9 null or
 * misaligned b, -10 ldb < max(1, m), -11 nrhs < 0.  n = 0 or nrhs = 0 is a no-op. */
int dhqr_solve_qrcp_f64(dhqr_handle h, int64_t m, int64_t n, int64_t rank, const double *dA, int64_t lda, const double *d_alpha,
                        const int64_t *d_jpvt, double *d_b, int64_t ldb, int nrhs, void *stream);

/* ---- host-buffer entry points (single GPU): the call a CPU-side user of qr! / \ makes -------
 * hA (m x n, lda) is copied to the device, factored, and copied back with alpha; blocks until
 * the result is in host memory.  With pinned host memory the call is a pipeline: the matrix goes up in
 * column chunks, the factorisation starts on the first one, every later chunk joins the trailing matrix
 * after a catch-up with the reflectors already finished, and finished panels travel back while later
 * ones are factored; only the first upload and the last download are exposed.  Same reflectors as
 * dhqr_qr_f64 on the resident matrix (every column receives every reflector once, in order). */
int dhqr_qr_host_f64(dhqr_handle h, int64_t m, int64_t n, double *hA, int64_t lda, double *h_alpha,
                     int nb);
/* The upload plan dhqr_qr_host_f64 would use for an m x n matrix with panels of nb columns (pure host logic, needs no device;
 * exposed for tests and for callers that want to size pinned staging buffers): chunk j = columns [bounds[j], bounds[j+1]),
 * j < *nchunks; join[j] = step of the look-ahead schedule at which it enters the trailing matrix (join[0] = 0: the first chunk is
 * the initial window).  Every boundary is a multiple of nb (the last is n); join is non-decreasing and never later than one step
 * before the panel chain reaches into the chunk (bounds[j] / nb - 3).  chunk, first, h2d_gbs, tflops, chain_us: the options
 * "host_chunk", "host_first", "host_h2d_gbs", "host_tflops", "host_chain_us".  cap = capacity of bounds (cap) and join (cap - 1). */
int dhqr_plan_host_upload(int64_t m, int64_t n, int nb, int chunk, int first, int h2d_gbs, int tflops, int chain_us, int cap,
                          int64_t *bounds, int *join, int *nchunks);
/* x = H \ b from a host-resident factorisation (hA, h_alpha) and host b (length m); x length n. */
int dhqr_ldiv_host_f64(dhqr_handle h, int64_t m, int64_t n, const double *hA, int64_t lda,
                       const double *h_alpha, const double *h_b, double *h_x);

/* ---- primitives exposed for parity tests ---------------------------------------------------- */
/* partialdot(a, b, is, ::Type{<:Real}) (S:42-49): *d_out = sum_{i in [i0,i1)} a[i]*b[i] (0-based). */
int dhqr_partialdot_f64(dhqr_handle h, const double *d_a, const double *d_b, int64_t i0, int64_t i1,
                        double *d_out, void *stream);
/* A[i,j] = U[0,1) from the counter-based generator keyed on (seed, i0+i, j0+j); bit-identical to
 * oracle/dhqr_oracle.c:dhqr_oracle_uniform (mirrors rand(T,m,n) at test/runtests.jl:45-46). */
int dhqr_fill_uniform_f64(dhqr_handle h, uint64_t seed, int64_t i0, int64_t j0, int64_t m, int64_t n,
                          double *dA, int64_t lda, void *stream);

/* ---- kernel-level hooks (unit tests of the individual CUDA kernels; not part of the drop-in) --
 * gemm_vta : Wext[nbp x (nbp+ncols)] = V' * [V | C]  (split over rows, partials reduced by ymake/tinv)
 * tinv     : Linv = (I + stril(V'V))^{-1}
 * ymake    : Y = -Linv * W
 * gemm_cvy : C += V * Y   on rows >= row_lo
 * All operate on the handle's internal V buffer, filled from (dV, ldv) by the call. */
int dhqr_k_block_reflector_f64(dhqr_handle h, int64_t rows, int nbp, const double *dV, int64_t ldv,
                               int64_t row_lo, int ncols, double *dC, int64_t ldc, double *d_linv_out,
                               void *stream);
/* Copy an internal workspace buffer ("wpart", "ybuf", "linv", "vbuf") to d_dst (debugging / tests). */
int dhqr_debug_copy_f64(dhqr_handle h, const char *which, double *d_dst, int64_t nelems, void *stream);
/* Panel kernel: factor the rows x ncols (ncols <= 32) panel at dP in place (reference recurrences
 * S:127-135 + S:208-209 restricted to the panel), alpha -> d_alpha[0:ncols]. */
int dhqr_k_panel_f64(dhqr_handle h, int64_t rows, int ncols, double *dP, int64_t ldp, double *d_alpha,
                     void *stream);

/* 128-column panel chain (CholeskyQR2 + Householder reconstruction, dhqr_wide.cuh): factor the rows x 128 panel at dP in
 * place (same output as 128 steps of S:127-135 + S:208-209 restricted to the panel), alpha -> d_alpha[0:128].
 * *refused = 1 when the on-device guards turned the panel down (dP is then untouched).  Synchronises `stream`. */
int dhqr_k_wide_panel_f64(dhqr_handle h, int64_t rows, double *dP, int64_t ldp, double *d_alpha, int *refused,
                          void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DHQR_H */
