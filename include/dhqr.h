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
 *     refused panel is redone by the 32-column chain), and so does dhqr_cod_f64, which factors R_r' on that path; (iii) with nranks > 1 every qr / apply_qt /
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
 *     re-entrant either: Polyester @batch, S:203-206).  Results are bitwise independent of what the handle ran before and of
 *     other handles at work on the same device (tests/test_gpu_history.py holds every entry point to this).
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
 * Distributed/SharedArrays (S:116-118, S:141-143, S:227-229, S:260-267, S:302, S:318).
 * NCCL is loaded on first use (here or in dhqr_nccl_unique_id): from the path in the environment variable
 * DHQR_NCCL_LIBRARY if it is set (opened RTLD_LOCAL, so it never displaces a libnccl the process already has), otherwise
 * libnccl.so.2 by soname.
 * Both create calls write *h only on success; a failed call leaves *h as it was and holds nothing on the device. */
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
 *   "profile"     1: CUDA-event bracket around every kernel launch (implies serial), read with dhqr_profile_get: the
 *                 classes together count every launch that dhqr_launch_count counts while it is on
 *   "bs_wave", "unblocked_wave", "fuse_house"  1 (default): back-substitution (and the Float64 forward substitution of
 *                 dhqr_forwardsolve_f64 / dhqr_solve_adj_f64) as one wavefront launch per right-hand side where all its CTAs fit
 *                 on the device, nb = 1 as one persistent launch (m <= 8192), nb = 1 with the next reflector formed inside the
 *                 apply kernel, where the shape allows; 0: the per-block / per-column launches those paths otherwise take
 *   "wide_kappa"  guard of the 128-column chain on ||D R1^{-1}||_F of its first Cholesky factor (default 1000)
 *   traces:       "panel_trace", "la_trace", "wide_trace" (timestamps read with dhqr_debug_copy_f64); "chain_wait_trace" 1:
 *                 under the look-ahead schedule, CUDA events around every launch on the chain's streams and %globaltimer
 *                 stamps of its first CTA start and last warp end ("chain_wait": [0] = launches, then per launch unit,
 *                 stream (0 chain, 1 second apply, 2 side kernels), class index for dhqr_profile_get, event span, stamp
 *                 span, their difference, in ms; -1 for a launch without stamps); "gemm_trace" 1: zero the rows and trace every
 *                 later k_gemm_vta / k_gemm_cvy_p launch, one row of 8 words per CTA (kind = (1 << 16) | NBP for k_gemm_vta,
 *                 (2 << 16) | K for k_gemm_cvy_p; then the clock64 cycles its MMA warps spent from entry to the first operand
 *                 stage, waiting on later stages, in the k-loop body, waiting on the C tile, in the epilogue, after the last
 *                 DMMA or epilogue, and from entry to exit, each summed over the warps), 0: stop, keep the rows ("gemm_trace":
 *                 [0] = rows, [1] = launches left untraced once the 2^17 rows are used, then the rows; synchronise first)
 *   "epoch_near_wrap" 1 (test hook, write-only): move the 32-bit launch-tag counters of the panel exchange cells (k_panel,
 *                 k_tp_panel), the wavefront substitutions and the nb = 1 wave to two launches below their resets, so that a short
 *                 test crosses the resets a long-lived handle meets after ~10^8 panel or ~4 x 10^9 wave launches.  Changes no result
 *                 and nothing else; takes effect on tag buffers the handle already has (one allocated later starts over at 0)
 *   read-only:    "sms", "rank", "nranks", "panels_fast", "panels_fallback" (inner panels taken by either path; device-side
 *                 counters of work the device has finished: read them after synchronising the stream of the calls),
 *                 "wide_panels" (outer panels factored by the 128-column chain), "wide_redone" (restarts after a refusal),
 *                 "qrcp_renorms" (exact column renorms of dhqr_qrcp_f64 and dhqr_qrcp_c64; device-side, read after synchronising),
 *                 "append_max_rows" (the largest k one dhqr_qr_append_f64 call takes on this device), "batch_max_elems" (the
 *                 largest m * n of one problem of the batched entry points, and the largest k (n + nrhs) of the batched append and
 *                 downdate), "batch_update_max_cols" (the largest n + nrhs of the batched append and downdate, and the largest n of
 *                 dhqr_backsolve_batched_f64)
 *   dhqr_get_option reads "nb", "panel_ctas", "sync", "profile", "lookahead", "panel_fast", "wide_panel", "cvy_persist",
 *                 "qt_vec", "bs_wave", "unblocked_wave", "fuse_house", "host_chunk" and the read-only keys (not "epoch_near_wrap").
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
 *     otherwise a multiple of 32 in [32,128].
 * The blocked paths (nb != 1) take m <= 728 x min(SMs, 160) rows (the 32-column panel kernel keeps its slab of rows in shared
 * memory; read-only option "append_max_rows") and return -2 beyond that, with A untouched; nb = 1 has no row limit. */
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

/* ---- complete orthogonal decomposition on the pivoted QR (not in the reference; LAPACK dgelsy's minimum-norm solution) --------
 * From A P = Q R (dhqr_qrcp_f64) at rank r: R_r = rows [0, r) of R = triu(A, 1) + diag(alpha), an r x n upper trapezoid, and the
 * unpivoted QR of its transpose, R_r' = Z [U; 0], give A P ~ Q1 [U' 0] Z' (DESIGN §2.8).  Float64, single GPU (a handle with
 * nranks > 1 returns -1), stream-ordered.  Every pointer must be 8 B aligned; every check runs before anything is enqueued.
 *
 * dhqr_cod_f64: F (n x rank, ldf >= max(1, n)) <- the factorisation of R_r' = Z [U; 0] in the library's storage format, gamma (rank)
 * <- diag(U).  A and alpha are read, never written; nothing outside F's n x rank block and gamma is written.  The factorisation is
 * the one dhqr_qr_f64 runs for nb = 0 on F, with the handle's options, so it synchronises the stream once when a 128-column panel of
 * R_r' went through the speculative wide chain (point (ii)).  n = 0 or rank = 0 is a no-op.  Errors: -1 null or multi-rank handle,
 * -2 m < 0, -3 n < 0 or n > m, or n above the row limit of the blocked unpivoted path (R_r' has n rows), -4 rank < 0 or rank > n,
 * -5 null or misaligned A, -6 lda < max(1, m), -7 null or misaligned alpha, -8 F null (rank > 0), misaligned, or overlapping A's
 * m x n block or alpha, -9 ldf < max(1, n), -10 gamma null (rank > 0), misaligned, or overlapping A, alpha or F. */
int dhqr_cod_f64(dhqr_handle h, int64_t m, int64_t n, int64_t rank, const double *dA, int64_t lda, const double *d_alpha,
                 double *dF, int64_t ldf, double *d_gamma, void *stream);
/* x = P Z [U^{-T} (Q'b)[0:rank]; 0]: the minimum-norm solution of the rank-`rank` problem min ||Q1 R_r P' x - b||, from
 * dhqr_qrcp_f64's (A, jpvt) and dhqr_cod_f64's (F, gamma) at the same rank.  d_b: m x nrhs, ldb >= max(1, m), in place: on return
 * b[0:n] = x, and rows n..m-1 hold rows n..m-1 of H_rank ... H_1 b, as in dhqr_solve_qrcp_f64.  rank = 0 gives x = 0.  jpvt
 * entries outside [0, n) are skipped.  No synchronisation apart from workspace growth (point (iv)).  Errors: -1 to -6 as above,
 * -7 null or misaligned jpvt, -8 F null (rank > 0) or misaligned, -9 ldf < max(1, n), -10 gamma null (rank > 0) or misaligned,
 * -11 null or misaligned b, -12 ldb < max(1, m), -13 nrhs < 0.  n = 0 or nrhs = 0 is a no-op. */
int dhqr_solve_cod_f64(dhqr_handle h, int64_t m, int64_t n, int64_t rank, const double *dA, int64_t lda, const int64_t *d_jpvt,
                       const double *dF, int64_t ldf, const double *d_gamma, double *d_b, int64_t ldb, int nrhs, void *stream);

/* ---- ComplexF64 QR with column pivoting and the complete orthogonal decomposition (LAPACK zgeqp3 + zgelsy) --------------------
 * The twins of dhqr_qrcp_f64, dhqr_solve_qrcp_f64, dhqr_cod_f64 and dhqr_solve_cod_f64, argument for argument, with void* for
 * ComplexF64 data (DESIGN §2.9).  Single GPU (a handle with nranks > 1 returns -1), n <= m, no row limit.  Stream-ordered; no call
 * synchronises apart from workspace growth (point (iv)); dhqr_cod_c64 factors R_r^H on the complex unpivoted path, which never
 * synchronises, so it has no point (ii).  Two calls on the same input give bitwise identical results.  Nothing outside the
 * documented operands is written.  Every ComplexF64 pointer (A, alpha, F, gamma, b) must be 16 B aligned: one that is only 8 B
 * aligned returns minus its argument index before anything is enqueued; jpvt stays int64_t*, 8 B aligned.  Every check runs
 * before anything is enqueued.  Error numbering is that of the Float64 twin.
 *
 * dhqr_qrcp_c64: factors in place.  On return (dA, lda, d_alpha) is the factorisation of A[:, jpvt] in the library's complex storage
 * format (v scaled to ||v||^2 = 2, H_j = I - v_j v_j^H, complex alpha), so dhqr_apply_qt_c64, dhqr_backsolve_c64, dhqr_form_q_c64,
 * dhqr_forwardsolve_c64 and dhqr_solve_adj_c64 take it as that.  Pivots as in dhqr_qrcp_f64 (largest partial norm, ties to the
 * smallest index, a NaN norm beats every number).  alpha_k = -exp(i angle(x0)) ||x||, formed as dhqr_qr_c64 forms it, signed-zero
 * pivots included.  Once the largest remaining norm is exactly 0, every remaining step stores v = 0 and alpha = 0 (H = I).  Exact
 * renorms count in the read-only option "qrcp_renorms".  Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 null
 * (n > 0) or misaligned A, -5 lda < max(1, m), -6 null or misaligned alpha, -7 null or misaligned jpvt.  n = 0 is a no-op. */
int dhqr_qrcp_c64(dhqr_handle h, int64_t m, int64_t n, void *dA, int64_t lda, void *d_alpha, int64_t *d_jpvt, void *stream);
/* x = P [R11^{-1} (Q^H b)[0:rank]; 0], the basic solution at the given rank, from dhqr_qrcp_c64.  d_b: m x nrhs, ldb >= max(1, m),
 * in place: on return b[0:n] = x, and rows n..m-1 hold rows n..m-1 of H_rank ... H_1 b.  rank = 0 gives x = 0.  jpvt entries outside
 * [0, n) are skipped.  Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 rank < 0 or rank > n, -5 null or
 * misaligned A, -6 lda < max(1, m), -7 null or misaligned alpha, -8 null or misaligned jpvt, -9 null or misaligned b,
 * -10 ldb < max(1, m), -11 nrhs < 0.  n = 0 or nrhs = 0 is a no-op. */
int dhqr_solve_qrcp_c64(dhqr_handle h, int64_t m, int64_t n, int64_t rank, const void *dA, int64_t lda, const void *d_alpha,
                        const int64_t *d_jpvt, void *d_b, int64_t ldb, int nrhs, void *stream);
/* dhqr_cod_c64: F (n x rank, ldf >= max(1, n)) <- the factorisation of R_r^H = Z [U; 0] (a conjugating transpose of the leading rank
 * rows of R) in the library's complex storage format, gamma (rank) <- diag(U), complex.  A and alpha are read, never written; nothing
 * outside F's n x rank block and gamma is written.  The factorisation is the one dhqr_qr_c64 runs.  n = 0 or rank = 0 is a no-op.
 * Errors: -1 null or multi-rank handle, -2 m < 0, -3 n < 0 or n > m, -4 rank < 0 or rank > n, -5 null or misaligned A,
 * -6 lda < max(1, m), -7 null or misaligned alpha, -8 F null (rank > 0), misaligned, or overlapping A's m x n block or alpha,
 * -9 ldf < max(1, n), -10 gamma null (rank > 0), misaligned, or overlapping A, alpha or F.  No row-limit error: the complex path has
 * no row limit. */
int dhqr_cod_c64(dhqr_handle h, int64_t m, int64_t n, int64_t rank, const void *dA, int64_t lda, const void *d_alpha, void *dF,
                 int64_t ldf, void *d_gamma, void *stream);
/* x = P Z [U^{-H} (Q^H b)[0:rank]; 0], the minimum-norm solution at the given rank, from dhqr_qrcp_c64's (A, jpvt) and
 * dhqr_cod_c64's (F, gamma) at the same rank.  d_b as in dhqr_solve_qrcp_c64.  rank = 0 gives x = 0.  jpvt entries outside [0, n)
 * are skipped.  Errors: -1 to -6 as above, -7 null or misaligned jpvt, -8 F null (rank > 0) or misaligned, -9 ldf < max(1, n),
 * -10 gamma null (rank > 0) or misaligned, -11 null or misaligned b, -12 ldb < max(1, m), -13 nrhs < 0.  n = 0 or nrhs = 0 is a
 * no-op. */
int dhqr_solve_cod_c64(dhqr_handle h, int64_t m, int64_t n, int64_t rank, const void *dA, int64_t lda, const int64_t *d_jpvt,
                       const void *dF, int64_t ldf, const void *d_gamma, void *d_b, int64_t ldb, int nrhs, void *stream);

/* ---- triangular-pentagonal QR: fold new rows into a factorisation (not in the reference; LAPACK dtpqrt / dtpmqrt) -----------
 * [R; B] = Q~ [R'; 0] (DESIGN §2.10): R = triu(dR[0:n, 0:n], 1) + diag(alpha) is the n x n triangle of any factorisation in the
 * library's storage format (dR may be the factored matrix itself), B the k x n block of new rows (ldb >= max(1, k)).  Only the strict
 * upper triangle of dR's n x n block is read and written: its diagonal and lower trapezoid (the original reflectors) are never
 * touched, so the original factorisation stays valid for dhqr_apply_qt_f64.  On return R' is in dR's strict upper triangle and in
 * alpha; Q~ = H~_1 ... H~_n with H~_j = I - v~_j v~_j', v~_j = vtop[j] on row j of the R block and B[:, j] on the k new rows,
 * ||v~_j||^2 = 2 or 0: B is overwritten with the reflector tails V2, vtop (length n) with their tops.  Each column follows the
 * recurrences of dhqr_qr_f64 on the stacked (n + k) x n matrix, alpha_j = -sign(x0) ||x|| with x0 = R[j, j] in its current state and
 * a zero x0 counted as positive (as in dhqr_qrcp_f64); a zero column stores v~ = 0 and alpha = 0.  In exact arithmetic R' is the R
 * of the stacked factorisation.  Least squares needs no further entry point: x = R'^{-1} c is dhqr_backsolve_f64(h, n, n, 0, n, dR,
 * ldr, alpha, c, ldc, nrhs, stream), which reads R's strict upper triangle and alpha only.
 * Single GPU (a handle with nranks > 1 returns -1).  Stream-ordered, no synchronisation apart from workspace growth (point (iv)).
 * Two calls on the same input give bitwise identical results, independent of ldr, ldb and 8 B base offsets.  Nothing outside the
 * documented operands is written.  k is capped by the slab capacity of the panel kernel, the row limit of the blocked dhqr_qr_f64
 * (728 x min(SMs, 160) rows; read-only option "append_max_rows"): a larger block returns -3 and is split by the caller.  n = 0 or
 * k = 0 is a no-op.  Every check runs before anything is enqueued.  Errors: -1 null or multi-rank handle, -2 n < 0, -3 k < 0 or
 * above the cap, -4 null (n > 0) or misaligned R, -5 ldr < max(1, n), -6 null or misaligned alpha, -7 null, misaligned B, or B
 * overlapping R's n x n block or alpha, -8 ldb < max(1, k), -9 null or misaligned vtop, or vtop overlapping R, alpha or B. */
int dhqr_qr_append_f64(dhqr_handle h, int64_t n, int64_t k, double *dR, int64_t ldr, double *d_alpha, double *dB, int64_t ldb,
                       double *d_vtop, void *stream);
/* [c; e] <- Q~' [c; e] (dhqr_apply_qt_append_f64) or Q~ [c; e] (dhqr_apply_q_append_f64), from (B, vtop) of dhqr_qr_append_f64:
 * c is n x nrhs (ldc >= max(1, n)), e is k x nrhs (lde >= max(1, k)), both in place.  T is recomputed from V2.  Same stream and
 * determinism rules.  n = 0, k = 0 or nrhs = 0 is a no-op.  Errors: -1 to -3 as above, -4 null or misaligned B, -5 ldb < max(1, k),
 * -6 null or misaligned vtop, -7 null or misaligned c, or c overlapping B or vtop, -8 ldc < max(1, n), -9 null or misaligned e, or
 * e overlapping B, vtop or c, -10 lde < max(1, k), -11 nrhs < 0. */
int dhqr_apply_qt_append_f64(dhqr_handle h, int64_t n, int64_t k, const double *dB, int64_t ldb, const double *d_vtop,
                             double *d_c, int64_t ldc, double *d_e, int64_t lde, int nrhs, void *stream);
int dhqr_apply_q_append_f64(dhqr_handle h, int64_t n, int64_t k, const double *dB, int64_t ldb, const double *d_vtop,
                            double *d_c, int64_t ldc, double *d_e, int64_t lde, int nrhs, void *stream);

/* ---- downdate: delete rows from a factorisation (not in the reference; LINPACK dchdd, scipy qr_delete, MATLAB qrdelete) -------
 * Theta [R; Z] = [R'; 0] with R''R' = R'R - Z'Z (DESIGN §2.11): R as for dhqr_qr_append_f64, Z the k x n block of rows to remove
 * (ldz >= max(1, k)).  Theta = Theta_n ... Theta_1, Theta_j = I - v~_j v~_j' J with J = diag(I_n, -I_k), v~_j = vtop[j] on row j of the
 * R block and Z[:, j] on the k rows, v~_j' J v~_j = 2 or 0.  Theta is J-orthogonal (Theta' J Theta = J), not orthogonal.  Column j
 * with x0 = R[j, j] in its current state and t = ||Z[:, j]||^2: sigma^2 = (|x0| - sqrt(t)) (|x0| + sqrt(t)), alpha_j = -sign(x0) sigma
 * (a zero x0 counted as positive); a zero column (x0 = 0, t = 0) stores v~ = 0 and alpha = 0.  The same storage contract as the
 * append: only R's strict upper triangle and alpha are read and written, Z is overwritten with V2 and vtop with the tops.
 * The caller is responsible for removing only rows that were folded in.  The library detects only the impossible cases: the first
 * column with sigma^2 <= 0 while t > 0 (R'R - Z'Z is not positive definite: the rows were never in A, or their removal leaves a
 * rank-deficient matrix), or with a NaN sigma^2.  Its 1-based index goes to *d_info (int64_t, device memory), and that column and
 * every later one store vtop = 0, V2 = 0 and alpha = NaN (Theta_j = I); rows of R' above it are the exact downdate of those rows.
 * Otherwise *d_info = 0.  *d_info is zero-filled in stream order before the first panel and written on the device, so reading it
 * is the caller's synchronisation.  n = 0 or k = 0 is a no-op that writes nothing, d_info included.  Single GPU, stream-ordered,
 * bitwise deterministic and layout-independent as the append, with the same cap on k ("append_max_rows", -3 above it).
 * Errors: -1 to -9 as for dhqr_qr_append_f64 with Z in place of B, -10 null (n > 0 and k > 0) or misaligned info, or info
 * overlapping R, alpha, Z or vtop. */
int dhqr_qr_downdate_f64(dhqr_handle h, int64_t n, int64_t k, double *dR, int64_t ldr, double *d_alpha, double *dZ, int64_t ldz,
                         double *d_vtop, int64_t *d_info, void *stream);
/* [c; e] <- Theta [c; e], Theta = Theta_n ... Theta_1, from (Z, vtop) of dhqr_qr_downdate_f64: with c = (Q'b)[0:n] and e the
 * right-hand sides of the removed rows, c' = the first n rows of the result gives x' = R'^{-1} c', and the residual sum of squares
 * drops by ||e'||^2.  No inverse apply is provided: Theta applied in reverse column order is its own inverse.  Operands, stream and
 * determinism rules and errors as for dhqr_apply_qt_append_f64, with Z in place of B. */
int dhqr_apply_downdate_f64(dhqr_handle h, int64_t n, int64_t k, const double *dZ, int64_t ldz, const double *d_vtop,
                            double *d_c, int64_t ldc, double *d_e, int64_t lde, int nrhs, void *stream);

/* ---- batched QR of many small problems (not in the reference; cuBLAS geqrfBatched / gelsBatched, torch.geqrf on a batch) --------
 * Problem i (0-based, i < batch) is the m x n column-major matrix at dA + i * stride_a (leading dimension lda), its alpha is at
 * d_alpha + i * stride_alpha (n entries) and its right-hand sides at d_b + i * stride_b (m x nrhs, ldb).  Float64, single GPU (a
 * handle with nranks > 1 returns -1).  One launch factors, applies or solves the whole batch (DESIGN §2.12): each problem is held in
 * the shared memory of one thread-block cluster of 1, 2, 4 or 8 CTAs, chosen from (m, n) alone.
 *   - Size limit: n <= m and m * n <= batch_max_elems (read-only option; 196 608 = 8 CTAs x 24 576 doubles, e.g. 8192 x 24,
 *     4096 x 48, 443 x 443).  A larger problem returns -3: there is no fall-back to dhqr_qr_f64, which takes it.
 *   - Strides: when batch > 1, stride_a >= lda * n, stride_alpha >= n and stride_b >= ldb * nrhs (ignored when batch <= 1).  The span
 *     of A over the batch must not intersect the span of alpha or of b (an interval test); batch x (CTAs per problem) <= 2^31 - 1.
 *   - Stream-ordered on the caller's stream.  No synchronisation and no allocation, ever: the batched entry points use no handle
 *     workspace, so they capture into a CUDA graph on a fresh handle.  Each call is one kernel launch (dhqr_launch_count; profile
 *     classes k_qr_batched, k_apply_qt_batched, k_apply_q_batched, k_solve_batched).
 *   - Bitwise deterministic: a problem's bits depend on its own data and on (m, n, nrhs) only, not on batch, its position in the
 *     batch, lda, ldb, the strides, 8 B base offsets or the handle's history.  Nothing outside the operands is written: neither
 *     padding rows nor the gaps between problems.
 *   - Errors, in argument order, every check before anything is enqueued: -1 null or multi-rank handle, -2 m < 0, -3 n < 0, n > m
 *     or m * n above batch_max_elems, -4 batch < 0 or too large for the grid, -5 null (batch > 0 and n > 0) or misaligned A, -6 lda
 *     < max(1, m), -7 stride_a < lda * n with batch > 1; then, at their own indices, null, misaligned (8 B) or overlapping alpha /
 *     b, stride_alpha < n, ldb < max(1, m), stride_b < ldb * nrhs and nrhs < 0.  batch = 0, n = 0 or nrhs = 0 is a no-op that
 *     writes nothing.
 *
 * dhqr_qr_batched_f64: factors every problem in place into the library's storage format (v scaled to |v|^2 = 2 in the lower
 * trapezoid including the diagonal, R's strict upper triangle above it, diag(R) in alpha), by the reference's recurrences as
 * oracle/dhqr_oracle.c and dhqr_qr_f64 with nb = 1 follow them, sign(0) = 0 included: an exact zero column gives the fp64 oracle's
 * NaN pattern.  So every other entry point reads problem i as a factorisation (dhqr_form_q_f64, dhqr_backsolve_f64,
 * dhqr_solve_adj_f64, ... on dA + i * stride_a).  The bits need not equal dhqr_qr_f64's: the sums run in another order.
 * Errors past -7: -8 null, misaligned or overlapping alpha, -9 stride_alpha < n. */
int dhqr_qr_batched_f64(dhqr_handle h, int64_t m, int64_t n, int64_t batch, double *dA, int64_t lda, int64_t stride_a,
                        double *d_alpha, int64_t stride_alpha, void *stream);
/* b <- Q'b (dhqr_apply_qt_batched_f64) or Q b (dhqr_apply_q_batched_f64) of every problem, for any nrhs >= 0.  Errors past -7:
 * -8 null, misaligned or overlapping b, -9 ldb < max(1, m), -10 stride_b < ldb * nrhs, -11 nrhs < 0. */
int dhqr_apply_qt_batched_f64(dhqr_handle h, int64_t m, int64_t n, int64_t batch, const double *dA, int64_t lda,
                              int64_t stride_a, double *d_b, int64_t ldb, int64_t stride_b, int nrhs, void *stream);
int dhqr_apply_q_batched_f64(dhqr_handle h, int64_t m, int64_t n, int64_t batch, const double *dA, int64_t lda,
                             int64_t stride_a, double *d_b, int64_t ldb, int64_t stride_b, int nrhs, void *stream);
/* Least squares, Q'b and the back-substitution fused in one launch: on return b[0:n] = x = R^{-1} (Q'b)[0:n], and rows n..m-1 hold
 * rows n..m-1 of Q'b, so the residual norm of each right-hand side is ||b[n:m]||.  A zero alpha propagates Inf / NaN, as in
 * dhqr_backsolve_f64.  Errors past -7: -8 null, misaligned or overlapping alpha, -9 stride_alpha < n, -10 null, misaligned or
 * overlapping b (A or alpha), -11 ldb < max(1, m), -12 stride_b < ldb * nrhs, -13 nrhs < 0. */
int dhqr_solve_batched_f64(dhqr_handle h, int64_t m, int64_t n, int64_t batch, const double *dA, int64_t lda, int64_t stride_a,
                           const double *d_alpha, int64_t stride_alpha, double *d_b, int64_t ldb, int64_t stride_b, int nrhs,
                           void *stream);

/* ---- batched append and downdate: rows into and out of many small triangles (not in the reference; DESIGN §2.13) -------------
 * Problem i: R = triu(dR_i[0:n, 0:n], 1) + diag(alpha_i) with dR_i = dR + i * stride_r (leading dimension ldr >= max(1, n); any
 * factorisation in the library's storage format, e.g. a problem of dhqr_qr_batched_f64), alpha_i = d_alpha + i * stride_alpha, the
 * k x n block B_i (or Z_i) at dB + i * stride_b (ldb >= max(1, k)), vtop_i = d_vtop + i * stride_vtop (n entries), and, when
 * nrhs > 0, c_i = d_c + i * stride_c (n x nrhs, ldc >= max(1, n)) and e_i = d_e + i * stride_e (k x nrhs, lde >= max(1, k)).
 * Per problem, the storage contract is that of dhqr_qr_append_f64 / dhqr_qr_downdate_f64: only R's strict upper triangle and alpha
 * are read and written, B (Z) is overwritten with the reflector tails V2 and vtop receives their tops, so dhqr_apply_qt_append_f64 /
 * dhqr_apply_downdate_f64 take (B_i, vtop_i) unchanged.  [c_i; e_i] is transformed in the same launch (Q~'[c; e] for the append,
 * Theta [c; e] for the downdate); nrhs = 0 transforms nothing, and c and e may then be null.  Each column follows the single-problem
 * recurrences: alpha_j = -sign(x0) ||x|| with a zero x0 counted as positive (not dhqr_qr_batched_f64's sign(0) = 0), a zero column
 * stores v~ = 0 and alpha = 0; the downdate's sigma^2 = (|x0| - sqrt(t)) (|x0| + sqrt(t)) and its failure rule: the first column with
 * sigma^2 <= 0 while t > 0, or a NaN sigma^2, goes 1-based into d_info[i] (int64_t, batch entries, contiguous; 0 when the problem's
 * removal succeeded), and that column and every later one of problem i store vtop = 0, V2 = 0, alpha = NaN.
 *   - One cluster of 1, 2, 4 or 8 CTAs per problem, chosen from (n, k, nrhs) alone; the slab of [B | e] stays in shared memory and R
 *     is read and written row by row.  Size limit: n + nrhs <= batch_update_max_cols (read-only option; 1024) and k (n + nrhs) <=
 *     batch_max_elems (196 608), so that the slab (at most 24 576 + n + nrhs doubles per CTA) and three vectors of n + nrhs doubles
 *     fit the 227 KiB of shared memory a CTA can have.  A larger block returns -3 and is split by the caller.
 *   - Single GPU (a handle with nranks > 1 returns -1), stream-ordered, one kernel launch per call (profile classes
 *     k_append_batched, k_downdate_batched), no workspace, no allocation, no synchronisation: a call captures into a CUDA graph on a
 *     fresh handle.  Bitwise deterministic: a problem's bits depend on its own data and on (n, k, nrhs) only, not on batch, its
 *     position, the leading dimensions, the strides, 8 B base offsets or the handle's history.  Nothing outside the operands is
 *     written.  batch = 0, n = 0 or k = 0 is a no-op that writes nothing, d_info included.
 *   - Strides (batch > 1): stride_r >= ldr * n, stride_alpha >= n, stride_b >= ldb * n, stride_vtop >= n, stride_c >= ldc * nrhs,
 *     stride_e >= lde * nrhs.  The span of every operand over the batch must not intersect the span of an earlier one.
 *   - Errors, in argument order, every check before anything is enqueued: -1 null or multi-rank handle, -2 n < 0, -3 k < 0 or the
 *     size limit, -4 batch < 0 or batch x (CTAs per problem) > 2^31 - 1, -5 null (batch > 0, n > 0) or misaligned R, -6 ldr < max(1, n),
 *     -7 stride_r, -8 null, misaligned or overlapping alpha, -9 stride_alpha, -10 null (batch, n, k > 0), misaligned or overlapping B,
 *     -11 ldb < max(1, k), -12 stride_b, -13 null, misaligned or overlapping vtop, -14 stride_vtop; with nrhs > 0: -15 null, misaligned
 *     or overlapping c, -16 ldc < max(1, n), -17 stride_c, -18 null, misaligned or overlapping e, -19 lde < max(1, k), -20 stride_e;
 *     -21 nrhs < 0; the downdate: -22 null, misaligned or overlapping info. */
int dhqr_qr_append_batched_f64(dhqr_handle h, int64_t n, int64_t k, int64_t batch, double *dR, int64_t ldr, int64_t stride_r,
                               double *d_alpha, int64_t stride_alpha, double *dB, int64_t ldb, int64_t stride_b, double *d_vtop,
                               int64_t stride_vtop, double *d_c, int64_t ldc, int64_t stride_c, double *d_e, int64_t lde, int64_t stride_e,
                               int nrhs, void *stream);
int dhqr_qr_downdate_batched_f64(dhqr_handle h, int64_t n, int64_t k, int64_t batch, double *dR, int64_t ldr, int64_t stride_r,
                                 double *d_alpha, int64_t stride_alpha, double *dZ, int64_t ldz, int64_t stride_z, double *d_vtop,
                                 int64_t stride_vtop, double *d_c, int64_t ldc, int64_t stride_c, double *d_e, int64_t lde,
                                 int64_t stride_e, int nrhs, int64_t *d_info, void *stream);
/* b_i[0:n] <- R_i^{-1} b_i[0:n] for every problem: R_i = triu(dR_i, 1) + diag(alpha_i) as above (only the strict upper triangle and
 * alpha are read; the diagonal and lower part of dR_i may hold anything), b_i = d_b + i * stride_b (n x nrhs, ldb >= max(1, n); rows
 * below n are neither read nor written).  The back-substitution of dhqr_solve_batched_f64, one CTA per problem and chunk of up to
 * 32 right-hand sides; n <= batch_update_max_cols.  A zero alpha propagates Inf / NaN.  Same stream, graph, determinism and no-op
 * rules (profile class k_backsolve_batched).  Errors: -1 null or multi-rank handle, -2 n < 0 or n > batch_update_max_cols, -3
 * batch < 0 or > 2^31 - 1, -4 null (batch > 0, n > 0) or misaligned R, -5 ldr < max(1, n), -6 stride_r < ldr * n, -7 null or
 * misaligned alpha, -8 stride_alpha < n, -9 null, misaligned or overlapping (R, alpha) b, -10 ldb < max(1, n), -11 stride_b < ldb *
 * nrhs, -12 nrhs < 0.  batch = 0, n = 0 or nrhs = 0 is a no-op. */
int dhqr_backsolve_batched_f64(dhqr_handle h, int64_t n, int64_t batch, const double *dR, int64_t ldr, int64_t stride_r,
                               const double *d_alpha, int64_t stride_alpha, double *d_b, int64_t ldb, int64_t stride_b, int nrhs,
                               void *stream);

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
/* Copy an internal workspace buffer ("wpart", "ybuf", "linv", "vbuf") to d_dst (debugging / tests).  "epochs": the three
 * launch-tag counters (panel cells, wavefronts, nb = 1 wave) as doubles, copied synchronously. */
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
