/* b200lops.h -- C ABI of libb200lops.so
 *
 * H100-native (sm_90a) kernels + NCCL collectives for the pylops-mpi
 * distributed matvec/rmatvec hot path.  Plain pointers and sizes only: every
 * buffer is a raw DEVICE pointer owned by the caller (unless a parameter is
 * explicitly named *_host), every stream is a cudaStream_t passed as void*.
 * Every entry point returns 0 on success, a cudaError_t (1..999) on a CUDA
 * failure, 1000+ncclResult_t on an NCCL failure, or a B2_ERR_* code; none
 * throws, none frees or retains caller memory past the call (handles such as
 * b2_ctx / b2_comm own their private workspaces and have *_destroy).
 *
 * Each declaration cites the reference interface (file:line relative to
 * pylops_mpi/ of PyLops/pylops-mpi @ fb5b7d4) it replaces.
 */
#ifndef B200LOPS_H
#define B200LOPS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_VERSION 100

/* element types */
enum { B2_F32 = 0, B2_F64 = 1, B2_C64 = 2, B2_C128 = 3, B2_BF16 = 4, B2_I64 = 5 };
/* reduction operators (mpi4py MPI.SUM / MPI.MAX / MPI.MIN, utils/_nccl.py:23-43) */
enum { B2_SUM = 0, B2_MAX = 1, B2_MIN = 2 };
/* local part of DistributedArray._compute_vector_norm, DistributedArray.py:688-758 */
enum { B2_NRM_COUNT_NONZERO = 0, B2_NRM_SUM_ABS = 1, B2_NRM_SUM_SQ = 2,
       B2_NRM_MAX_ABS = 3, B2_NRM_MIN_ABS = 4, B2_NRM_SUM_POW = 5 };
/* MPIFirstDerivative kinds, basicoperators/FirstDerivative.py:104-127 */
enum { B2_FD_FORWARD = 0, B2_FD_BACKWARD = 1, B2_FD_CENTERED = 2 };
/* op(A) for gemv/gemm */
enum { B2_OP_N = 0, B2_OP_T = 1, B2_OP_H = 2 };
enum { B2_THRESH_NONE = 0, B2_THRESH_SOFT = 1, B2_THRESH_HARD = 2, B2_THRESH_HALF = 3 };
/* curve kinds of b2_radon (pylops.signalprocessing.Radon2D / Radon3D kind=) */
enum { B2_RADON_LINEAR = 0, B2_RADON_PARABOLIC = 1, B2_RADON_HYPERBOLIC = 2 };

/* error codes >= 2000 are library-level */
enum { B2_OK = 0, B2_ERR_DTYPE = 2001, B2_ERR_ARG = 2002, B2_ERR_HALO = 2003,
       B2_ERR_WORKSPACE = 2004, B2_ERR_UNSUPPORTED = 2005, B2_ERR_ALIGN = 2006, B2_ERR_CONVERGE = 2007 };

/* per-device context: SM count + the reduction workspace (per-CTA partials, ticket counter) shared by b2_dot /
 * b2_norm_partial / b2_dot_multi / b2_sparse_update / the transposed b2_gemv.  Calls that use the workspace must be
 * stream-ordered with respect to each other: use one b2_ctx per stream that issues reductions concurrently.
 * Every workspace address stays valid until b2_ctx_destroy, so a CUDA graph may capture calls that use it: the
 * transposed b2_gemv's chunk-partial scratch only grows, keeps each buffer it outgrows until b2_ctx_destroy and never
 * synchronises; when it would have to grow while the stream is capturing, b2_gemv returns B2_ERR_WORKSPACE and
 * enqueues nothing (run the call once eagerly before capturing it).  Destroy the graphs before the context. */
typedef struct b2_ctx b2_ctx;
typedef struct b2_comm b2_comm;          /* one NCCL communicator (world, mask group, grid row / col) */
typedef struct b2_mailbox b2_mailbox;    /* peer-memory mailboxes: one-shot collectives and the fused halo exchange */

int b2_version(void);
const char* b2_strerror(int code);

/* ---- context --------------------------------------------------------- */
int b2_ctx_create(int device, b2_ctx** out);
int b2_ctx_destroy(b2_ctx* ctx);
int b2_ctx_sm_count(const b2_ctx* ctx, int* out);

/* ---- element-wise (DistributedArray.py:574-652, 809-837: add, iadd,
 *      multiply, __neg__, conj, copy, zeros_like) ------------------------- */
/* out = a * op(x) + b * y ; a,b are (re,im) host pairs; y may be NULL (b ignored);
 * op = conj when conj_x != 0.  out may alias x or y. */
int b2_lincomb(b2_ctx* ctx, void* out, const double a[2], const void* x, const double b[2],
               const void* y, size_t n, int dtype, int conj_x, void* stream);
/* Same with DEVICE-resident real scalars: a = a_scale * (*a_dev) (a_dev may be NULL -> 1),
 * b likewise; lets a solver iteration run with no host round-trip
 * (optimization/cls_basic.py:389-397 does five .item() syncs per iteration). */
int b2_lincomb_dev(b2_ctx* ctx, void* out, const double* a_dev, double a_scale, const void* x,
                   const double* b_dev, double b_scale, const void* y, size_t n, int dtype,
                   void* stream);
/* b2_lincomb_dev fused with the reduction the CGLS recurrence needs next: out = a x + b y (real device scalars) and
 * norm2_dev[0] = sum |out|^2 (float64, local partial; norm2_dev[1] = 0 for complex dtypes so that the caller's
 * (re, im) slot layout is kept).  x.x after x += a c, s.s after s -= a q, c.c after c = r + b c
 * (cls_basic.py:389-401): one pass and one launch each instead of two.  Shares the ctx reduction workspace. */
int b2_lincomb_dev_norm2(b2_ctx* ctx, void* out, const double* a_dev, double a_scale, const void* x,
                         const double* b_dev, double b_scale, const void* y, size_t n, int dtype,
                         double* norm2_dev, void* stream);
/* out = op(x) * y element-wise (DistributedArray.multiply, :630-652) */
int b2_mul(b2_ctx* ctx, void* out, const void* x, const void* y, size_t n, int dtype,
           int conj_x, void* stream);
int b2_fill(b2_ctx* ctx, void* out, const double v[2], size_t n, int dtype, void* stream);

/* ---- local reductions (the per-rank half of DistributedArray.dot :654-686
 *      and _compute_vector_norm :688-758); results are float64 in DEVICE
 *      memory, accumulated in float64 in a fixed (deterministic) order ----- */
/* out_dev[0..1] = sum_i op(x_i) * y_i  (re, im); op = conj when conj_x (numpy.vdot) */
int b2_dot(b2_ctx* ctx, const void* x, const void* y, size_t n, int dtype, int conj_x,
           double* out_dev, void* stream);
/* out_dev[0] = local partial for the requested norm kind (p only for SUM_POW).  A NaN element makes every kind but
 * COUNT_NONZERO return NaN, MAX_ABS and MIN_ABS included (as np.max / np.linalg.norm); COUNT_NONZERO counts it. */
int b2_norm_partial(b2_ctx* ctx, const void* x, size_t n, int dtype, int kind, double p,
                    double* out_dev, void* stream);
/* axis-wise variant (DistributedArray.norm(ord, axis=...), DistributedArray.py:688-758, 796-807): x is the local block
 * viewed as [n_outer][n_axis][n_inner]; out_dev[o * n_inner + i] = float64 partial over the middle axis for the same
 * norm kinds and the same NaN rule as b2_norm_partial (the caller combines partials across ranks when the axis is the
 * partition axis and takes the root); n_axis == 0 writes each kind's identity (0, or +inf for MIN_ABS) */
int b2_norm_axis(b2_ctx* ctx, const void* x, size_t n_outer, size_t n_axis, size_t n_inner, int dtype, int kind,
                 double p, double* out_dev, void* stream);
/* k dot products <x_j, y_j> in ONE launch: out_dev[0..k) for real dtypes, out_dev[0..2k) as
 * (re, im) pairs for complex dtypes (CGLS needs q.q and c.c
 * together, r.r / s.s / x.x together -- cls_basic.py:389, 394-401) */
int b2_dot_multi(b2_ctx* ctx, int k, const void* const* xs, const void* const* ys, size_t n,
                 int dtype, int conj_x, double* out_dev, void* stream);

/* out = |num / (den1 + alpha * den2)| on DEVICE scalars (den2 may be NULL): the CGLS step length
 * a = kold / (q.q + damp c.c) and ratio b = k / kold (cls_basic.py:389, 395) with no host sync */
int b2_scalar_div(double* out_dev, const double* num_dev, const double* den1_dev,
                  const double* den2_dev, double alpha, void* stream);

/* Device-side history of solver scalars: hist[it * nvals + j] = |src[j * stride]| (skipped when it >= cap), then the
 * optional scalar copy *copy_dst = *copy_src (kold <- k, cls_basic.py:397) and ++(*it_dev) (uint64).  With it a block of
 * CGLS iterations (cls_basic.py:370-404) needs no host synchronisation and can be replayed as a CUDA graph. */
int b2_history_push(const double* src_dev, int nvals, int stride, double* hist_dev, void* it_dev, size_t cap,
                    double* copy_dst_dev, const double* copy_src_dev, void* stream);

/* ---- LSQR (optimization/cls_basic.py LSQR; the definition is scipy.sparse.linalg.lsqr, Paige & Saunders 1982) ----
 * The solver state is one float64 DEVICE array of B2_LSQR_NSTATE doubles at these offsets.  BB / DD and AA are the
 * (all-reduced) reductions the kernels read: BB = |U|^2 (complex dtypes: BB+1 = 0, as b2_lincomb_dev_norm2 writes it),
 * DD = |dk|^2 of the previous update, AA = |V|^2.  u and v are kept unnormalised (U = u', V = v' of lsqr.py, norms
 * beta and alfa); the coefficient slots fold scipy's normalisations into the next combination:
 *   U <- INV_ALFA * (A V) - CUB * U      V <- CVA * (A^H U) - CVB * V       (b2_lincomb_dev_norm2, b scale -1)
 * The host fills the constants and the state after scipy's initialisation; every other slot is the kernels'. */
enum { B2_LSQR_BB = 0, B2_LSQR_DD = 2, B2_LSQR_AA = 4,
       B2_LSQR_ALFA = 8, B2_LSQR_BETA, B2_LSQR_RHOBAR, B2_LSQR_PHIBAR, B2_LSQR_ANORM, B2_LSQR_DDNORM, B2_LSQR_RES2,
       B2_LSQR_XXNORM, B2_LSQR_Z, B2_LSQR_CS2, B2_LSQR_SN2, B2_LSQR_ITN, B2_LSQR_ISTOP, B2_LSQR_PENDING,
       B2_LSQR_STOPPED,
       B2_LSQR_DAMP = 24, B2_LSQR_DAMPSQ, B2_LSQR_ATOL, B2_LSQR_BTOL, B2_LSQR_CTOL, B2_LSQR_BNORM, B2_LSQR_ITER_LIM,
       B2_LSQR_R1NORM = 32, B2_LSQR_R2NORM, B2_LSQR_ACOND, B2_LSQR_ARNORM, B2_LSQR_XNORM, B2_LSQR_TEST1,
       B2_LSQR_TEST2, B2_LSQR_TT1, B2_LSQR_RTOL,
       B2_LSQR_CUB = 42, B2_LSQR_CVA, B2_LSQR_CVB,
       B2_LSQR_T1 = 48, B2_LSQR_T2, B2_LSQR_INV_RHO, B2_LSQR_INV_ALFA,     /* b2_lsqr_update's coef_dev */
       B2_LSQR_SCRATCH = 52, B2_LSQR_NSTATE = 56,
       B2_LSQR_HIST = 9 /* history row: r1norm r2norm anorm acond arnorm xnorm test1 test2 istop */ };
/* One scalar step of lsqr.py's loop, one thread, scipy's operations in scipy's order with round-to-nearest intrinsics
 * (csrc/lsqr.cu writes the sequence out), so the state equals a float64 NumPy transcription bit for bit.
 *   phase 0 (after BB, DD are reduced): finish the pending iteration -- ddnorm += DD, acond, test3, istop, history
 *           row itn-1 into hist_dev[(itn-1) * B2_LSQR_HIST ...] when itn-1 < cap, STOPPED = 1 if istop != 0 -- then
 *           beta = sqrt(BB) and the v-step coefficients CVA, CVB;
 *   phase 1 (after AA is reduced): itn += 1, anorm, alfa = sqrt(AA), the rotations, T1 / T2 / INV_RHO / INV_ALFA,
 *           the xnorm recurrence, r1norm, r2norm, arnorm, test1, test2, CUB; the iteration is then pending;
 *   phase 2: finish the pending iteration only (after the last iteration of a block; DD reduced).
 * Every phase is a no-op once STOPPED.  B2_ERR_ARG: null state, phase outside 0..2, null hist with cap > 0. */
int b2_lsqr_scalars(double* state_dev, int phase, double* hist_dev, size_t cap, void* stream);
/* LSQR model-side update in ONE pass (lsqr.py:467-476), coef_dev = state + B2_LSQR_T1 (t1, t2, inv_rho, inv_alfa):
 *   dk = inv_rho w;  x += t1 w;  var += dk^2 (var may be NULL: calc_var=False);  w = inv_alfa v + t2 w;
 *   *dd_dev = sum |dk|^2 (float64, local partial, deterministic last-CTA fold; shares the ctx reduction workspace).
 * Complex data are arrays of 2n reals except var += dk^2, NumPy's complex square (re = dr dr - di di, im = dr di +
 * di dr).  Products and sums are rounded in T one by one (no contraction).  16-byte accesses when x, w, v, var are
 * 16-byte aligned.  When stop_dev is non-NULL and *stop_dev != 0 nothing is written (the LSQR STOPPED slot).
 * B2_ERR_ARG: null ctx / coef / dd, or (n > 0) a null or aliased x, w, v, var; B2_ERR_DTYPE: not F32/F64/C64/C128. */
int b2_lsqr_update(b2_ctx* ctx, void* x, void* w, const void* v, void* var, size_t n, int dtype,
                   const double* coef_dev, const double* stop_dev, double* dd_dev, void* stream);

/* ---- ISTA / FISTA model update ("next" row; optimization/cls_sparsity.py:270-343, 578-662) in ONE pass:
 *   u = base + alpha*g (g may be NULL);  v = threshold_kind(u, thresh) (_apply_thresh, cls_sparsity.py:21-46);
 *   xnew = v;  znew = v + c*(v - xold) (znew may be NULL; FISTA's auxiliary model, :640-644);
 *   sums_dev[0] = sum|v - xold|^2 (0 if xold NULL), sums_dev[1] = sum|v| -- local partials of the update norm
 *   (:331) and the l1 cost (:333).  xnew/znew may alias base/xold.  HALF is real-only.  A NaN in u gives NaN in xnew
 *   under every kind (complex SOFT: both components), as pylops' NumPy thresholds do, and so NaN sums. */
int b2_sparse_update(b2_ctx* ctx, const void* base, const void* g, double alpha, const void* xold,
                     double thresh, int kind, void* xnew, void* znew, double c, double* sums_dev,
                     size_t n, int dtype, void* stream);

/* ---- MPIFirstDerivative per-rank apply (FirstDerivative.py:129-319) -------
 * x,y: this rank's row block [nrows_local x ncols] (C order) of the global
 * [nrows_global x ncols] array, global row offset row0.  halo_lo holds the n_lo
 * rows immediately before row0, halo_hi the n_hi rows immediately after the
 * block (the add_ghost_cells payload, DistributedArray.py:876-953); NULL / 0
 * at the global edges.  Complex arrays: pass the real dtype and 2*ncols.
 * B2_ERR_HALO, for this and b2_second_derivative alike, when n_lo / n_hi is less than the rows that the taps of
 * the block's own rows read below / above it.  That is at most the _halo reach, and no rows past a global edge. */
int b2_first_derivative(b2_ctx* ctx, const void* x, void* y, const void* halo_lo, int n_lo,
                        const void* halo_hi, int n_hi, size_t nrows_local, size_t ncols,
                        size_t row0, size_t nrows_global, int kind, int order, int edge,
                        double sampling, int adjoint, int dtype, void* stream);
/* rows below / above itself that any row of the stencil reads (0 to 2), the wider of edge = 0 and 1 */
int b2_first_derivative_halo(int kind, int order, int adjoint, int* need_lo, int* need_hi);
/* MPISecondDerivative per-rank apply (basicoperators/SecondDerivative.py:125-257): same contract as
 * b2_first_derivative (row block + up to 2 halo rows per side, exact-transpose adjoint, B2_ERR_HALO rule),
 * scale 1/sampling^2 */
int b2_second_derivative(b2_ctx* ctx, const void* x, void* y, const void* halo_lo, int n_lo,
                         const void* halo_hi, int n_hi, size_t nrows_local, size_t ncols, size_t row0,
                         size_t nrows_global, int kind, int edge, double sampling, int adjoint, int dtype,
                         void* stream);
/* rows below / above itself that any row of the stencil reads (0 to 2) */
int b2_second_derivative_halo(int kind, int edge, int adjoint, int* need_lo, int* need_hi);
/* rank-local first (deriv=1) / second (deriv=2) derivative along the MIDDLE axis of a C-ordered
 * [n_outer][n_axis][n_inner] block: the non-partitioned directions of MPILaplacian / MPIGradient
 * (Laplacian.py:97-126, Gradient.py:101-119 wrap a serial pylops derivative per rank) */
int b2_derivative_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                       int deriv, int kind, int order, int edge, double sampling, int adjoint, int dtype,
                       void* stream);
/* rank-local 1-D convolution along the MIDDLE axis of a C-ordered [n_outer][n_axis][n_inner] block with nh real
 * taps h (device pointer, same dtype as x); forward y[i] = sum_k h[k] x[i+offset-k], adjoint = exact transpose.
 * pylops.signalprocessing.Convolve1D inside MPIBlockDiag (tutorials/reflectivity.py:74-76).  dtype F32 / F64
 * (complex data: the real dtype and 2 * n_inner); 0 <= offset < nh, x != y; any nh is exact, nh > n_axis included */
int b2_convolve_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                     const void* h, int nh, int offset, int adjoint, int dtype, void* stream);
/* rank-local post-stack modelling along the MIDDLE axis of the same block: pylops.avo.poststack.
 * PoststackLinearModelling, y = C D x with D the first derivative along the axis (FirstDerivative, edge=False,
 * sampling=1, kind B2_FD_CENTERED or B2_FD_FORWARD) and C the convolution of b2_convolve_axis; adjoint x = D^T C^T y.
 * One launch; equals b2_derivative_axis then b2_convolve_axis (adjoint: the reverse) bit for bit.  Arguments and
 * error codes as b2_convolve_axis, plus B2_ERR_ARG for any other kind; y is untouched on every error */
int b2_poststack_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                      const void* h, int nh, int offset, int kind, int adjoint, int dtype, void* stream);
/* rank-local NON-STATIONARY 1-D convolution along the MIDDLE axis of the same block: pylops.signalprocessing.
 * NonStationaryConvolve1D.  hs is a device array [nfilt][nh] of real filters (the data's real dtype) at the axis
 * samples oh + dh * f; sample j uses h_j, interpolated linearly between its two neighbouring filters in float64
 * weights cast to the dtype (two rounded products, one rounded add), the first / last filter outside [oh, oh +
 * dh * (nfilt - 1)].  Forward y[i] = sum_j h_j[hc + i - j] x[j], adjoint = exact transpose, both summed in ascending
 * sample order with fma; no atomics, no allocation, repeated applies give identical bits.  dtype F32 / F64 (complex
 * data: the real dtype and 2 * n_inner).  B2_ERR_ARG: a null pointer, x == y, a zero size, nfilt < 1, nh < 1, hc
 * outside [0, nh), dh < 1; B2_ERR_DTYPE: another dtype; y is untouched on every error */
int b2_nsconvolve_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                       const void* hs, int nfilt, int nh, int hc, long long oh, long long dh, int adjoint, int dtype,
                       void* stream);
/* the 2-D wavelet branch of pylops.avo.poststack.PoststackLinearModelling: y = C D x with D as in b2_poststack_axis
 * and C the convolution of b2_nsconvolve_axis; adjoint x = D^T C^T y.  One launch; equals b2_derivative_axis then
 * b2_nsconvolve_axis (adjoint: the reverse) bit for bit.  Arguments and error codes as b2_nsconvolve_axis, plus
 * B2_ERR_ARG for a kind other than B2_FD_CENTERED / B2_FD_FORWARD */
int b2_nspoststack_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                        const void* hs, int nfilt, int nh, int hc, long long oh, long long dh, int kind, int adjoint,
                        int dtype, void* stream);
/* rank-local NON-STATIONARY 2-D convolution of a C-ordered [nx][nz][n_inner] image (n_inner 1, or 2 for complex data
 * as (re, im) pairs of the real dtype): pylops.signalprocessing.NonStationaryConvolve2D.  hs is a device array
 * [nfx][nfz][nhx][nhz] of real filters (the data's real dtype) at the points (ohx + dhx a, ohz + dhz b), centre
 * (nhx / 2, nhz / 2); point j uses h_j, bilinear in the bank with float64 per-axis weights (the first / last filter
 * outside the nodes), each weight product rounded to the dtype.  Forward y[i] = sum_j h_j[hc + i - j] x[j], adjoint =
 * exact transpose.  One launch, no atomics, no allocation: repeated applies give identical bits.  dtype F32 / F64.
 * B2_ERR_ARG: a null pointer, x == y, an empty image, n_inner not 1 or 2, nfx / nfz / nhx / nhz < 1, dhx / dhz < 1;
 * B2_ERR_DTYPE: another dtype; y is untouched on every error */
int b2_nsconvolve2d(b2_ctx* ctx, const void* x, void* y, size_t nx, size_t nz, size_t n_inner, const void* hs, int nfx,
                    int nfz, int nhx, int nhz, long long ohx, long long dhx, long long ohz, long long dhz, int adjoint,
                    int dtype, void* stream);
/* rank-local NON-STATIONARY FILTER ESTIMATION, adjoint: pylops.signalprocessing.NonStationaryFilters2D^H (and
 * NonStationaryFilters1D^H with nx = nfx = nhx = 1, ohx = 0, dhx = 1).  For a C-ordered real image d [nx][nz] and the
 * fixed real image inp [nx][nz], writes the bank hs_out [nfx][nfz][nhx][nhz] of the transpose of b2_nsconvolve2d's
 * forward in its bank: g_c[k] = sum_(j in S_c) W_c[j] inp[j] d[j + k - hc], with the points, weights, supports and
 * centres of b2_nsconvolve2d.  Each filter's support is split into a number of parts fixed by the shape; with more
 * than one part the partial banks go to work (b2_nsfilters2d_work_bytes bytes, 0 with one part) and are folded in
 * ascending order.  No atomics, no allocation: the bits depend only on the shape and the dtype.  dtype F32 / F64.
 * B2_ERR_ARG: a null ctx, d, inp or hs_out, hs_out overlapping d or inp, an empty image, an axis over 2^40 samples
 * or an image over 2^50, nfx / nfz / nhx / nhz < 1, dhx / dhz < 1, more CTAs than one grid holds, a null or short work
 * (when one is needed) or work overlapping d, inp or hs_out; B2_ERR_DTYPE: another dtype; hs_out is untouched on every error */
int b2_nsfilters2d_adjoint(b2_ctx* ctx, const void* d, const void* inp, void* hs_out, size_t nx, size_t nz, int nfx,
                           int nfz, int nhx, int nhz, long long ohx, long long dhx, long long ohz, long long dhz,
                           void* work, size_t work_bytes, int dtype, void* stream);
/* *bytes = the workspace b2_nsfilters2d_adjoint needs for this shape and dtype; error codes as that entry's shape
 * checks, plus B2_ERR_ARG for a null bytes */
int b2_nsfilters2d_work_bytes(size_t nx, size_t nz, int nfx, int nfz, int nhx, int nhz, long long ohx, long long dhx,
                              long long ohz, long long dhz, int dtype, size_t* bytes);
/* rank-local NON-STATIONARY 3-D convolution of a C-ordered [nx][ny][nz][n_inner] volume (n_inner 1, or 2 for complex
 * data as (re, im) pairs of the real dtype): pylops.signalprocessing.NonStationaryConvolve3D.  hs is a device array
 * [nfx][nfy][nfz][nhx][nhy][nhz] of real filters (the data's real dtype) at the points (ohx + dhx a, ohy + dhy b,
 * ohz + dhz e), centre (nhx / 2, nhy / 2, nhz / 2); point j uses h_j, trilinear in the bank with float64 per-axis
 * weights (the first / last filter outside the nodes), each weight product (wz wy) wx rounded once to the dtype.
 * Forward y[i] = sum_j h_j[hc + i - j] x[j], adjoint = exact transpose.  One launch, no atomics, no allocation:
 * repeated applies give identical bits.  dtype F32 / F64.
 * B2_ERR_ARG: a null pointer, x == y, an empty axis, n_inner not 1 or 2, nfx / nfy / nfz / nhx / nhy / nhz < 1,
 * dhx / dhy / dhz < 1, an axis, filter size or node position of 2^29 samples or more (the kernel indexes each axis
 * in 32 bits), more tiles than one grid holds; B2_ERR_DTYPE: another dtype; y is untouched on every error */
int b2_nsconvolve3d(b2_ctx* ctx, const void* x, void* y, size_t nx, size_t ny, size_t nz, size_t n_inner, const void* hs,
                    int nfx, int nfy, int nfz, int nhx, int nhy, int nhz, long long ohx, long long dhx, long long ohy,
                    long long dhy, long long ohz, long long dhz, int adjoint, int dtype, void* stream);
/* rank-local Kirchhoff demigration, spreading / stacking stage: pylops.waveeqprocessing.Kirchhoff (mode="analytic",
 * 2-D or 3-D, dynamic=False) before its wavelet convolution (run that as b2_convolve_axis on the [ns*nr][nt] traces).
 * Tables are float64 device arrays in the kernel's layout: trav_srcs [ns][ni], trav_recs [nr][ni] (a trace reads
 * contiguous image points).  Forward: x is the image [ni], y the traces [ns*nr][nt] (trace isrc*nr + irec), every
 * sample written; adjoint: the reverse.  Per pair q = (trav_srcs + trav_recs) / dt in float64 (one add, one IEEE
 * divide), it = trunc(q), d = q - it, used iff 0 <= it < nt - 1: forward y[it] += x (1-d), y[it+1] += x d; adjoint
 * y += x[it] (1-d) + x[it+1] d, in (isrc, irec) order: float64 adjoints equal pylops' loop bit for bit.  Deterministic
 * (no floating-point atomics), no allocation.  dtype F32 / F64 (index math always float64).  B2_ERR_ARG: a null
 * pointer, x == y, a zero size, dt not finite and positive; B2_ERR_DTYPE: another dtype; y is untouched on every
 * error */
int b2_kirchhoff(b2_ctx* ctx, const void* x, void* y, const double* trav_srcs, const double* trav_recs, size_t ni,
                 size_t ns, size_t nr, size_t nt, double dt, int adjoint, int dtype, void* stream);
/* b2_kirchhoff over the image points [i0, i0 + nc) of an [ni] image, with that chunk's tables trav_srcs [ns][nc],
 * trav_recs [nr][nc].  Forward: x is the whole image (x[i0 .. i0+nc) is read), y the traces, overwritten
 * (accumulate 0) or added into (accumulate 1); adjoint: x the traces, y the whole image, of which y[i0 .. i0+nc) is
 * written.  i0 must be a multiple of 32: then chunks tiling [0, ni), applied in ascending order with accumulate 0
 * for the first and 1 after, give b2_kirchhoff's result bit for bit in F32 and F64.  B2_ERR_ARG: as b2_kirchhoff,
 * plus nc = 0, i0 not a multiple of 32, i0 + nc > ni, accumulate not 0 / 1, accumulate 1 with adjoint; y is
 * untouched on every error */
int b2_kirchhoff_chunk(b2_ctx* ctx, const void* x, void* y, const double* trav_srcs, const double* trav_recs,
                       size_t ni, size_t i0, size_t nc, size_t ns, size_t nr, size_t nt, double dt, int adjoint,
                       int accumulate, int dtype, void* stream);
/* rank-local Radon transform: pylops.signalprocessing.Radon2D / Radon3D (Spread's per-sample tables).  Model x
 * [npy][npx][nt][n_inner], data [nhy][nhx][nt][n_inner] (n_inner 1, or 2 for complex data as (re, im) pairs of the
 * real dtype); forward x -> y is model -> data, adjoint the reverse.  hy, hx, py, px are float64 device arrays of the
 * unitless offsets (samples of dh) and slownesses (linear, parabolic) or velocities (hyperbolic); hy = py = NULL is
 * 2-D (nhy = npy = 1, no y term is formed).  For model sample (p, t0) and trace h, in float64 rounded to nearest
 * operation by operation: linear tdec = (t0 + px*hx) + py*hy, parabolic (t0 + px*(hx*hx)) + py*(hy*hy), hyperbolic
 * sqrt((t0*t0 + (hx/px)*(hx/px)) + (hy/py)*(hy/py)).  interp != 0: used iff 0 <= tdec < nt - 1, it = trunc(tdec),
 * d = tdec - it, forward y[h][it] += (1-d) x[p][t0], y[h][it+1] += d x[p][t0]; interp = 0: used iff
 * 0 <= tdec < nt, y[h][trunc(tdec)] += x[p][t0]; the adjoint is the exact transpose.  Sums are float64, rounded once
 * to the dtype: forward over (py, px, t0) ascending, adjoint over (hy, hx) ascending.  One launch, no atomics, no
 * allocation: repeated applies give identical bits.  dtype F32 / F64.  B2_ERR_ARG: a null pointer (hy / py excepted,
 * which are NULL together), x == y, a zero size, nhy or npy other than 1 in 2-D, an axis of 2^31 samples or more,
 * n_inner not 1 or 2, an unknown kind, more CTAs than one grid holds; B2_ERR_DTYPE: another dtype; y is untouched on
 * every error */
int b2_radon(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t nhy, size_t nhx, size_t npy,
             size_t npx, const double* hy, const double* hx, const double* py, const double* px, int kind, int interp,
             int adjoint, int dtype, void* stream);
/* b2_radon applied to every window of a section, with the tapered overlap-add of b2_sliding, in one launch: the
 * sliding-window Radon transform of pylops.signalprocessing.Sliding2D / Sliding3D over Radon2D / Radon3D.  The section
 * [n0][n1][nt][n_inner] holds nwins0 x nwins1 windows of nhy x nhx traces, window w = i0 * nwins1 + i1 starting at
 * trace (i0 * step0, i1 * step1); the model is [nwins0 * nwins1][npy][npx][nt][n_inner], one b2_radon model block per
 * window, on the window-local offsets hy, hx (2-D: hy = py = NULL, nhy = npy = 1).  tap is b2_sliding's table
 * [nwins0 * nwins1][nhy][nhx] in the dtype (NULL: no taper).  Forward x (model) -> y (section): each section sample
 * sums, as b2_sliding's fold, tap * v over the windows that hold its trace, v the window's b2_radon value (a float64
 * sum rounded once to the dtype); samples no window holds are 0.  Adjoint x (section) -> y (model): each window's
 * b2_radon stack of tap * d, the product rounded to the dtype.  Both directions equal b2_radon per window plus
 * b2_sliding bit for bit.  One launch, no atomics, no allocation.  dtype F32 / F64.  B2_ERR_ARG: b2_radon's, and
 * b2_sliding's window checks, more CTAs than one grid holds; B2_ERR_DTYPE: another dtype; y is untouched on every
 * error */
int b2_radon_windows(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t n0, size_t n1, size_t nhy,
                     size_t nhx, size_t npy, size_t npx, const double* hy, const double* hx, const double* py,
                     const double* px, int kind, int interp, size_t nwins0, size_t nwins1, size_t step0,
                     size_t step1, const void* tap, int adjoint, int dtype, void* stream);
/* tapered overlap-add: the combining stage of pylops.signalprocessing.Sliding2D / Sliding3D.  Windows
 * [nwins0][nwins1][nwin0][nwin1][nt][n_inner] (n_inner values per sample: 2 for the (re, im) pairs of complex data in
 * the real dtype), data [n0][n1][nt][n_inner]; window w = i0 * nwins1 + i1 starts at trace (i0 * step0, i1 * step1).
 * tap [nwins0 * nwins1][nwin0][nwin1] is one taper value per window trace in the dtype (NULL: no taper).  Forward
 * (fold) x = windows -> y = data: each sample is the sum over i0 ascending of the sum over i1 ascending of
 * tap * window over the windows that hold its trace, every product and sum rounded to the dtype; samples no window
 * holds are 0.  Adjoint (unfold) x = data -> y = windows: tap * data.  One launch, no atomics, no allocation.  dtype
 * F32 / F64.  B2_ERR_ARG: a null pointer (tap excepted), x == y, a zero size, an axis of 2^31 or more, windows that
 * leave the section, 2^62 or more values; B2_ERR_DTYPE: another dtype; y is untouched on every error */
int b2_sliding(b2_ctx* ctx, const void* x, void* y, size_t n0, size_t n1, size_t nt, size_t n_inner, size_t nwins0,
               size_t nwins1, size_t nwin0, size_t nwin1, size_t step0, size_t step1, const void* tap, int adjoint,
               int dtype, void* stream);
/* b2_radon applied to every patch of a section, with the tapered overlap-add of b2_patch, in one launch: the
 * time-space patch Radon transform of pylops.signalprocessing.Patch2D / Patch3D over Radon2D / Radon3D.  The section
 * [n0][n1][ns][n_inner] holds nwins0 x nwins1 x nwins2 patches of nhy x nhx traces and nt samples, patch
 * w = (i0 * nwins1 + i1) * nwins2 + i2 starting at (trace i0 * step0, trace i1 * step1, sample i2 * step2); the model
 * is [nwins0 * nwins1 * nwins2][npy][npx][nt][n_inner], one b2_radon model block per patch on patch-local time and
 * the patch-local offsets hy, hx (2-D: hy = py = NULL, nhy = npy = 1).  tap0, tap1, tap2 are b2_patch's per-axis
 * float64 tapers.  Forward x (model) -> y (section): each section sample sums, as b2_patch's fold, tap * v over the
 * patches that hold it, v the patch's b2_radon value at the patch-local sample (a float64 sum rounded once to the
 * dtype); samples no patch holds are 0.  Adjoint x (section) -> y (model): each patch's b2_radon stack of tap * d, the
 * product rounded to the dtype.  Both directions equal b2_radon per patch plus b2_patch bit for bit.  One launch, no
 * atomics, no allocation.  dtype F32 / F64.  B2_ERR_ARG: b2_radon's checks, b2_patch's window checks, more CTAs than
 * one grid holds; B2_ERR_DTYPE: another dtype; y is untouched on every error */
int b2_radon_patches(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t n0, size_t n1, size_t ns,
                     size_t nhy, size_t nhx, size_t npy, size_t npx, const double* hy, const double* hx,
                     const double* py, const double* px, int kind, int interp, size_t nwins0, size_t nwins1,
                     size_t nwins2, size_t step0, size_t step1, size_t step2, const double* tap0, const double* tap1,
                     const double* tap2, int adjoint, int dtype, void* stream);
/* tapered overlap-add of time-space patches: the combining stage of pylops.signalprocessing.Patch2D / Patch3D and
 * Sliding1D.  Windows [nwins0][nwins1][nwins2][nwin0][nwin1][nwin2][n_inner] (n_inner values per sample: 2 for the
 * (re, im) pairs of complex data in the real dtype), data [n0][n1][nt][n_inner]; window
 * w = (i0 * nwins1 + i1) * nwins2 + i2 starts at (trace i0 * step0, trace i1 * step1, sample i2 * step2).  tap0
 * [nwins0][nwin0], tap1 [nwins1][nwin1], tap2 [nwins2][nwin2] are float64 per-axis tapers (NULL: that axis is not
 * tapered); a window sample's taper is ((tap0 * tap1) * tap2) in float64 rounded once to the dtype.  Forward (fold)
 * x = windows -> y = data: each sample is the sum over i0 ascending of the sum over i1 ascending of the sum over i2
 * ascending of tap * window over the windows that hold it, every product and sum rounded to the dtype; samples no
 * window holds are 0.  Adjoint (unfold) x = data -> y = windows: tap * data.  One launch, no atomics, no allocation.
 * dtype F32 / F64.  B2_ERR_ARG: a null pointer (the tapers excepted), x == y, a zero size, an axis of 2^31 or more,
 * windows that leave the section, 2^62 or more values; B2_ERR_DTYPE: another dtype; y is untouched on every error */
int b2_patch(b2_ctx* ctx, const void* x, void* y, size_t n0, size_t n1, size_t nt, size_t n_inner, size_t nwins0,
             size_t nwins1, size_t nwins2, size_t nwin0, size_t nwin1, size_t nwin2, size_t step0, size_t step1,
             size_t step2, const double* tap0, const double* tap1, const double* tap2, int adjoint, int dtype,
             void* stream);
/* analytic (constant-velocity) traveltime table of pylops.waveeqprocessing.Kirchhoff, in b2_kirchhoff_chunk's
 * layout: table[p][j] = |grid point i0 + j - point p| / vel for p < n, j < nc (row stride nc).  Axes are float64
 * device arrays; y = NULL for 2-D (ny ignored), where the grid is meshgrid(x, z, indexing="ij") raveled,
 * ii = ix * nz + iz, and pts is [2][n] with rows (x, z); in 3-D meshgrid(y, x, z, indexing="ij"),
 * ii = (iy * nx + ix) * nz + iz, pts [3][n] with rows (y, x, z).  NumPy's operations in NumPy's order, rounded to
 * nearest: 2-D sqrt((x-px)*(x-px) + (z-pz)*(z-pz)) / vel, 3-D sqrt(((x-px)*(x-px) + (z-pz)*(z-pz)) + (y-py)*(y-py))
 * / vel, equal to the float64 NumPy table bit for bit.  No allocation.  B2_ERR_ARG: a null pointer (y excepted), a
 * zero size (ny when y is given), i0 + nc > ny * nx * nz; table is untouched on every error */
int b2_kirchhoff_tables(b2_ctx* ctx, const double* y, const double* x, const double* z, size_t ny, size_t nx,
                        size_t nz, const double* pts, size_t n, double vel, size_t i0, size_t nc, double* table,
                        void* stream);
/* eikonal traveltime tables for pylops.waveeqprocessing.Kirchhoff(mode="eikonal") in b2_kirchhoff's layout:
 * table[p][ii] (row stride ny * nx * nz, float64) is the first-arrival time from grid node idx_host[p] = (iy, ix, iz)
 * (a HOST array [n][3]) through the velocity model vel [ny][nx][nz] (float64, ii = (iy * nx + ix) * nz + iz; 2-D is
 * ny = 1) on a grid of spacings dy, dx, dz.  The values are the iterate after max_iter Jacobi steps of the
 * first-order Godunov upwind update written out in csrc/eikonal.cu (T = 0 at the node, +inf elsewhere at the start),
 * rounded to nearest operation by operation: equal bit for bit to its NumPy restatement.  work is a device buffer
 * of b2_eikonal_work_bytes(ny, nx, nz, n) bytes, 8-byte aligned; info_host, if not NULL, receives 4 host words: the
 * Jacobi steps that changed a value (capped at max_iter), the passes run, the (tile, point) blocks computed and the
 * blocks of all passes.  Reads the device several times (construction-time, not capturable).  No allocation.
 * B2_ERR_ARG: a null pointer (info_host excepted), a zero size or max_iter, a node outside the grid, a spacing that
 * is not finite and positive, a velocity that is not finite and positive (table is untouched on these);
 * B2_ERR_CONVERGE: the max_iter-th iterate is not the fixed point (table holds that iterate) */
int b2_eikonal_tables(b2_ctx* ctx, const double* vel, size_t ny, size_t nx, size_t nz, double dy, double dx,
                      double dz, const long long* idx_host, size_t n, size_t max_iter, double* table, void* work,
                      long long* info_host, void* stream);
/* bytes of b2_eikonal_tables' work buffer for n points on an ny x nx x nz grid, about (n + 1) * ny * nx * nz * 8
 * (one more iterate and the slowness); 0 for a zero or too large size */
size_t b2_eikonal_work_bytes(size_t ny, size_t nx, size_t nz, size_t n);
/* Peer-memory halo exchange fused INTO the stencil kernel (replaces the add_ghost_cells Send/Recv pairs of
 * DistributedArray.py:876-953 as used by FirstDerivative.py:221-247, 276-319 and SecondDerivative.py), on the halo
 * region of the mailboxes of b2_mailbox_create.  ONE launch per apply: the first CTAs push the boundary rows into the
 * neighbours' boxes over NVLink and publish a flag, the CTAs of the first / last row chunk run last and wait for it.
 * Collective: same call sequence on every rank of the handle, all on one stream; each rank must own >= 2 rows;
 * 2 * ncols * sizeof(dtype) must fit in halo_cap (B2_ERR_WORKSPACE).  deriv = 1 | 2 (first | second derivative). */
int b2_derivative_peer(b2_ctx* ctx, b2_mailbox* h, const void* x, void* y, size_t nrows_local, size_t ncols,
                       size_t row0, size_t nrows_global, int deriv, int kind, int order, int edge, double sampling,
                       int adjoint, int dtype, void* stream);
/* Same operator on HOST buffers (pageable or pinned).  x_host / y_host address the
 * GLOBAL [nrows_global x ncols] arrays (to_dist keeps the global array replicated on
 * every rank's host, DistributedArray.py:440-459); this call processes rows
 * [row_begin, row_end) and only touches rows [row_begin-2, row_end+2) of x_host and
 * [row_begin, row_end) of y_host.  Row chunks go through the device with H2D /
 * kernel / D2H overlapped on three streams.  This is the host-buffer plugin entry
 * the end-to-end benchmark times. */
int b2_first_derivative_host(b2_ctx* ctx, const void* x_host, void* y_host, size_t nrows_global,
                             size_t ncols, size_t row_begin, size_t row_end, int kind, int order,
                             int edge, double sampling, int adjoint, int dtype);

/* ---- dense per-rank matvec (the pylops.MatrixMult block inside MPIBlockDiag /
 *      MPIVStack, BlockDiag.py:127-129,139-141; VStack.py:129-131,144-145; and
 *      the M==1 tile product of MPIMatrixMult, MatrixMult.py:366-370,670) ----
 * y[m or n] = op(A[m x n, row-major, leading dim lda]) x ; dtype_a in
 * {F32,F64,C64,C128,BF16}; x,y have dtype_xy (BF16 A pairs with F32 x/y).  Any m and n; op T / H with more than
 * 128 rows uses the context's chunk-partial scratch (B2_ERR_WORKSPACE rule above). */
int b2_gemv(b2_ctx* ctx, const void* A, size_t lda, size_t m, size_t n, const void* x, void* y,
            int op, int dtype_a, int dtype_xy, void* stream);

/* ---- dense tile product on the tensor cores, wgmma (MPIMatrixMult with M>1,
 *      MatrixMult.py:663-670, 742-763): C[m x n] (+)= op(A) B, A,B bf16,
 *      C fp32, all row-major ------------------------------------------------ */
int b2_gemm_bf16(b2_ctx* ctx, const void* A, size_t lda, const void* B, size_t ldb, float* C,
                 size_t ldc, size_t m, size_t n, size_t k, int op_a, int accumulate,
                 void* stream);
/* Stationary-A MPIMatrixMult (round 2): A tiles are operator state and never move; per apply the small operand is
 * all-gathered (cast to bf16 on the fly) and the partial products are reduce-scattered by the GEMM epilogue itself.
 *   b2_cast_bf16_multi: float32 tile -> bfloat16, stored to ndst <= 8 destinations (local or IPC-mapped peers):
 *                       the X / Y panel broadcasts of MatrixMult.py:663-670, 742-763 as ONE read of the tile.
 *   b2_gemm_bf16_seg  : op(A) B on the tensor cores with the output columns cut into nseg <= 8 segments of seg_cols
 *                       (multiple of 32) columns, segment c written to segs_host[c] (leading dimension ldc) -- peer
 *                       GPUs' staging buffers, i.e. the reduce-scatter rides on the epilogue's NVLink stores.
 *   b2_sum_slots      : out[rows x cols] = sum_s slots[s * slot_stride + r * ld_in + c] in slot order. */
int b2_cast_bf16_multi(b2_ctx* ctx, const float* src, size_t ld_src, size_t rows, size_t cols,
                       void* const* dsts_host, int ndst, size_t ld_dst, void* stream);
int b2_gemm_bf16_seg(b2_ctx* ctx, const void* A, size_t lda, const void* B, size_t ldb, float* const* segs_host,
                     int nseg, size_t seg_cols, size_t ldc, size_t m, size_t n, size_t k, int op_a, void* stream);
int b2_sum_slots(b2_ctx* ctx, const float* slots, size_t slot_stride, int nslots, size_t ld_in, float* out,
                 size_t rows, size_t cols, void* stream);
/* generic SIMT tile product for the dtypes tensor cores do not serve
 * (f32/f64/c64/c128 parity cases of tests/test_matrixmult.py); any m, n, k, leading dimensions >= the row lengths */
int b2_gemm(b2_ctx* ctx, const void* A, size_t lda, const void* B, size_t ldb, void* C, size_t ldc,
            size_t m, size_t n, size_t k, int op_a, int accumulate, int dtype, void* stream);

/* ---- MPIFredholm1 per-rank batched product (Fredholm1.py:119-129, 147-167):
 *      y[s] = op(G[s]) x[s] for s < nsl ; G[s] is nx x ny, x[s] is (ny|nx) x nz */
int b2_batched_gemm(b2_ctx* ctx, const void* G, const void* x, void* y, size_t nsl, size_t nx,
                    size_t ny, size_t nz, int adjoint, int dtype, void* stream);

/* Fused product + all-gather over NVLink peer memory: the epilogue stores every output element to
 * y (local) and to the same offset of `npeers` peer buffers (IPC-mapped; peers_host[d] already points
 * at the position matching y).  Replaces product-then-Allgather of Fredholm1.py:122-132 by ONE kernel;
 * completion across ranks = any stream-ordered collective after it (e.g. a 1-element b2_allreduce). */
int b2_batched_gemm_allgather(b2_ctx* ctx, const void* G, const void* x, void* y, void* const* peers_host,
                              int npeers, size_t nsl, size_t nx, size_t ny, size_t nz, int adjoint,
                              int dtype, void* stream);
/* Tensor-core (wgmma) plan for the same product, float32 / complex64 only (Fredholm1.py:119-129, 147-167).
 * G is operator state: plan creation splits G and G^H (the reference's `saveGt`, :105-106) ONCE into two fp16
 * planes each ("fp16x2": v*2^e = hi + lo*2^-11 with a power-of-two scale 2^e per output row, 22 significant
 * bits, three MMAs per k-step -> float32-class accuracy on the fp16 tensor pipe); complex64 runs as one real
 * product over the (re,im)-interleaved views.  b2_fredholm_apply packs x (one small kernel, which also takes a
 * power-of-two scale per column of x) and runs the batched product; with npeers > 0 the epilogue also stores
 * every output element to the same offset of the peers' IPC-mapped buffers (fused Allgather of Fredholm1.py:131-132,
 * completion = any stream-ordered cross-rank barrier after it).  The plan owns its device workspaces; applies
 * of one plan must be stream-ordered.  G must stay valid only during b2_fredholm_plan_create. */
typedef struct b2_fredholm_plan b2_fredholm_plan;
int b2_fredholm_plan_create(b2_ctx* ctx, const void* G, size_t nsl, size_t nx, size_t ny, size_t nz, int dtype,
                            b2_fredholm_plan** out);
int b2_fredholm_plan_destroy(b2_fredholm_plan* plan);
int b2_fredholm_apply(b2_fredholm_plan* plan, const void* x, void* y, void* const* peers_host, int npeers,
                      int adjoint, void* stream);
/* peer-mappable device buffers (cudaMalloc) and CUDA IPC handle plumbing (64-byte handles) */
int b2_symm_alloc(size_t bytes, void** out);
int b2_symm_free(void* p);
int b2_ipc_get_handle(void* p, void* handle64_host);
int b2_ipc_open_handle(const void* handle64_host, void** out);
int b2_ipc_close_handle(void* p);

/* Peer-memory mailboxes over NVLink (no NCCL): every rank of a group of 1..8 owns one box of
 * b2_mailbox_bytes(halo_cap) bytes (b2_symm_alloc), and boxes_host[r] is rank r's box as IPC-mapped in this process
 * (own pointer for r == rank).  The box has one region per use: the scalar all-reduce, the vector all-reduce /
 * all-gather, and the halo exchange of b2_derivative_peer, whose slots hold halo_cap bytes (a multiple of 16) per
 * parity and side.  Create zeroes this rank's region headers: every rank creates its handle before any rank's first
 * call on it.  Calls of each use keep a sequence number in device memory, so they can be captured in a CUDA graph;
 * the calls on one handle are collective and issued on one stream.  B2_ERR_ARG: a null pointer, size outside 1..8,
 * rank outside [0, size), halo_cap zero or not a multiple of 16. */
size_t b2_mailbox_bytes(size_t halo_cap);
int b2_mailbox_create(int rank, int size, void* const* boxes_host, size_t halo_cap, b2_mailbox** out);
int b2_mailbox_destroy(b2_mailbox* h);

/* One-shot all-reduce of k <= 8 float64 scalars: the collective half of DistributedArray.dot / norm
 * (DistributedArray.py:684-686, 714-757) and of the CGLS step scalars. */
int b2_peer_allreduce(b2_mailbox* h, double* vals_dev, int k, int op, void* stream);

/* One-shot SUM all-reduce of a small vector (<= b2_peer_vec_max_bytes()): the array Allreduce of
 * MPIVStack._rmatvec (VStack.py:146-148) / MatrixMult.py:420-426 in the latency regime. */
size_t b2_peer_vec_max_bytes(void);
int b2_peer_vec_allreduce(b2_mailbox* h, void* buf_dev, size_t n, int dtype, void* stream);

/* One-shot Allgather(v) (every chunk <= b2_peer_vec_max_bytes()): recv = concatenation of the ranks' counts_host[r]
 * elements.  The latency-regime replacement of the pad-to-max NCCL gather of utils/_nccl.py:363-403 (e.g. the
 * 128 KB model vector of MPIMatrixMult's single-column apply). */
int b2_peer_vec_allgatherv(b2_mailbox* h, const void* send, void* recv, const size_t* counts_host, int dtype,
                           void* stream);

/* ---- NCCL collectives (utils/_nccl.py:98-403, utils/_mpi.py:21-344,
 *      Distributed.py:35-349) --------------------------------------------- */
int b2_get_unique_id(void* id128_host);                       /* _nccl.py:98-132 */
int b2_comm_create(int rank, int size, const void* id128_host, int device, b2_comm** out);
int b2_comm_split(b2_comm* comm, int color, int key, b2_comm** out);   /* _nccl.py:135-165 */
int b2_comm_destroy(b2_comm* comm);
int b2_comm_rank(const b2_comm* comm, int* rank, int* size);
int b2_allreduce(b2_comm* comm, const void* send, void* recv, size_t n, int dtype, int op,
                 void* stream);                               /* _nccl.py:203-240 */
int b2_allgather(b2_comm* comm, const void* send, void* recv, size_t n_per_rank, int dtype,
                 void* stream);                               /* _nccl.py:167-200 */
/* uneven gather without the reference's pad-to-max (_nccl.py:363-403): rank r
 * contributes counts[r] elements; recv is the plain concatenation */
int b2_allgatherv(b2_comm* comm, const void* send, void* recv, const size_t* counts_host,
                  int dtype, void* stream);
/* same, with explicit placement: rank r's counts[r] elements land at recv + offsets[r] (elements);
 * send may alias its own destination (in-place). */
int b2_allgatherv_at(b2_comm* comm, const void* send, void* recv, const size_t* counts_host,
                     const size_t* offsets_host, int dtype, void* stream);
int b2_bcast(b2_comm* comm, void* buf, size_t n, int dtype, int root, void* stream);  /* :243-262 */
int b2_send(b2_comm* comm, const void* buf, size_t n, int dtype, int peer, void* stream); /* :265-286 */
int b2_recv(b2_comm* comm, void* buf, size_t n, int dtype, int peer, void* stream);       /* :289-316 */
int b2_group_start(void);
int b2_group_end(void);

#ifdef __cplusplus
}
#endif
#endif /* B200LOPS_H */
