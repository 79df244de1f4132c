// Dense per-rank matvec y = op(A) x  (the pylops.MatrixMult block applied by
// MPIBlockDiag / MPIVStack: pylops_mpi/basicoperators/BlockDiag.py:127-129,
// 139-141; VStack.py:129-131,144-145; and the single-RHS tile product of
// MPIMatrixMult, MatrixMult.py:366-370, 670).
//
// Single right-hand side => 0.5..1 flop per byte of A => HBM-bound; tensor cores
// do not apply.  Algorithmic bytes = m*n*sizeof(A) (+ vectors).
//  * op = N : one warp per row, 16-byte loads along the row, 4 in flight per lane,
//            x served from L1/L2, warp-shuffle reduction.
//  * op = T/H: one lane per 16-byte column vector, warps stride over the rows of a
//            row chunk, CTA-level smem fold, chunk partials folded in chunk order
//            by the last CTA of each column tile (deterministic, no atomics on y).
#include <limits.h>
#include "common.cuh"

namespace {

// ---- element traits ---------------------------------------------------------
template <typename TA> struct ElemTraits {   // float / double
  using X = TA; using Acc = TA; static constexpr int V = 16 / sizeof(TA);
  __device__ static __forceinline__ Acc zero() { return TA(0); }
  __device__ static __forceinline__ void fma_(Acc& acc, TA a, TA x, bool) { acc = fma(a, x, acc); }
  __device__ static __forceinline__ Acc add(Acc a, Acc b) { return a + b; }
};
template <typename R> struct ElemTraits<b2_cx<R>> {
  using X = b2_cx<R>; using Acc = b2_cx<R>; static constexpr int V = 16 / sizeof(b2_cx<R>);
  __device__ static __forceinline__ Acc zero() { return {R(0), R(0)}; }
  __device__ static __forceinline__ void fma_(Acc& acc, X a, X x, bool conj) {
    b2_cx_fma(acc, conj ? b2_cx_conj(a) : a, x);
  }
  __device__ static __forceinline__ Acc add(Acc a, Acc b) { return b2_cx_add(a, b); }
};
template <> struct ElemTraits<__nv_bfloat16> {
  using X = float; using Acc = float; static constexpr int V = 8;
  __device__ static __forceinline__ Acc zero() { return 0.f; }
  __device__ static __forceinline__ void fma_(Acc& acc, __nv_bfloat16 a, float x, bool) {
    acc = fmaf(__bfloat162float(a), x, acc);
  }
  __device__ static __forceinline__ Acc add(Acc a, Acc b) { return a + b; }
};

template <typename A> __device__ __forceinline__ A shfl_xor_t(A v, int o) { return __shfl_xor_sync(0xffffffffu, v, o); }
template <typename R> __device__ __forceinline__ b2_cx<R> shfl_xor_t(b2_cx<R> v, int o) {
  return {__shfl_xor_sync(0xffffffffu, v.re, o), __shfl_xor_sync(0xffffffffu, v.im, o)};
}

template <typename TA>
struct AVec {  // 16 bytes of A
  TA v[ElemTraits<TA>::V];
};
template <typename TA>
__device__ __forceinline__ AVec<TA> load_a(const TA* p) {
  uint4 r = ldg_stream16(p);
  AVec<TA> o;
  *reinterpret_cast<uint4*>(&o) = r;
  return o;
}

// cached scalar loads for every element type (a complex element in one 8- / 16-byte load)
template <typename T> __device__ __forceinline__ T ldg_t(const T* p) { return __ldg(p); }
template <typename R> __device__ __forceinline__ b2_cx<R> ldg_t(const b2_cx<R>* p) {
  const b2_pair_t<R> t = __ldg(reinterpret_cast<const b2_pair_t<R>*>(p));
  return {t.x, t.y};
}
template <typename T> __device__ __forceinline__ T ldcg_t(const T* p) { return __ldcg(p); }
template <typename R> __device__ __forceinline__ b2_cx<R> ldcg_t(const b2_cx<R>* p) {
  const b2_pair_t<R> t = __ldcg(reinterpret_cast<const b2_pair_t<R>*>(p));
  return {t.x, t.y};
}

template <typename TA>
struct XVec {  // the x elements matching one 16-byte vector of A
  typename ElemTraits<TA>::X v[ElemTraits<TA>::V];
};
template <typename TA>
__device__ __forceinline__ XVec<TA> load_x(const typename ElemTraits<TA>::X* p) {
  XVec<TA> o;
  constexpr int NQ = sizeof(XVec<TA>) / 16;
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4* d = reinterpret_cast<uint4*>(&o);
#pragma unroll
  for (int i = 0; i < NQ; ++i) d[i] = __ldg(q + i);
  return o;
}

// -------------------------------------------------------------------------
// op = N : y_i = sum_j A_ij x_j
// -------------------------------------------------------------------------
constexpr int GN_WARPS = 8;
constexpr int GN_UNROLL = 4;

template <typename TA, bool VEC>
__global__ void __launch_bounds__(GN_WARPS * 32)
gemv_n_kernel(const TA* __restrict__ A, size_t lda, size_t m, size_t n,
              const typename ElemTraits<TA>::X* __restrict__ x,
              typename ElemTraits<TA>::X* __restrict__ y) {
  using Tr = ElemTraits<TA>;
  using Acc = typename Tr::Acc;
  constexpr int V = Tr::V;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t row = (size_t)blockIdx.x * GN_WARPS + warp;
  if (row >= m) return;
  const TA* a = A + row * lda;
  Acc acc[GN_UNROLL];
#pragma unroll
  for (int u = 0; u < GN_UNROLL; ++u) acc[u] = Tr::zero();
  size_t j = 0;
  if (VEC) {
    const size_t nvec = n / V;
    size_t v = lane;
    for (; v + (GN_UNROLL - 1) * 32 < nvec; v += GN_UNROLL * 32) {
      AVec<TA> av[GN_UNROLL];
#pragma unroll
      for (int u = 0; u < GN_UNROLL; ++u) av[u] = load_a(a + (v + u * 32) * V);
#pragma unroll
      for (int u = 0; u < GN_UNROLL; ++u) {
        XVec<TA> xv = load_x<TA>(x + (v + u * 32) * V);
#pragma unroll
        for (int e = 0; e < V; ++e) Tr::fma_(acc[u], av[u].v[e], xv.v[e], false);
      }
    }
    for (; v < nvec; v += 32) {
      AVec<TA> av = load_a(a + v * V);
      XVec<TA> xv = load_x<TA>(x + v * V);
#pragma unroll
      for (int e = 0; e < V; ++e) Tr::fma_(acc[0], av.v[e], xv.v[e], false);
    }
    j = nvec * V;
  }
  for (size_t jj = j + lane; jj < n; jj += 32) Tr::fma_(acc[0], a[jj], x[jj], false);
  Acc s = Tr::add(Tr::add(acc[0], acc[1]), Tr::add(acc[2], acc[3]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = Tr::add(s, shfl_xor_t(s, o));
  if (lane == 0) y[row] = s;
}


// Long rows (>= 32 KB): with one warp per row a warp streams its whole row alone, so the kernel ends with a long
// tail in which the last few hundred warps run latency-bound (measured on 32768-column bf16 panels: a fixed ~40 us
// on top of bytes / bandwidth -- 0.94 of the HBM peak at 32768 rows, 0.84 at 16384, ~0.65 at 8192).  Here the 8 warps
// of a CTA sweep R rows TOGETHER, each warp taking every 8th 512-byte piece of all R rows: 2 R independent 16-byte
// loads per lane in flight, every x vector loaded once per R rows, work per CTA R rows instead of 8 -- a shorter,
// steeper tail.  Partial sums meet in shared memory and are added in warp order (deterministic).
constexpr int GS_WARPS = 8;
template <typename TA, int R>
__global__ void __launch_bounds__(GS_WARPS * 32)
gemv_n_split_kernel(const TA* __restrict__ A, size_t lda, size_t m, size_t n,
                    const typename ElemTraits<TA>::X* __restrict__ x,
                    typename ElemTraits<TA>::X* __restrict__ y) {
  using Tr = ElemTraits<TA>;
  using Acc = typename Tr::Acc;
  constexpr int V = Tr::V;
  constexpr size_t STEP = GS_WARPS * 32;
  __shared__ Acc part[GS_WARPS][R];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t row0 = (size_t)blockIdx.x * R;
  const TA* a[R];
  Acc acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const size_t row = row0 + r < m ? row0 + r : m - 1;     // rows past the end re-read the last row; never stored
    a[r] = A + row * lda;
    acc[r] = Tr::zero();
  }
  const size_t nvec = n / V;
  size_t v = (size_t)warp * 32 + lane;
  for (; v + STEP < nvec; v += 2 * STEP) {
    AVec<TA> a0[R], a1[R];
#pragma unroll
    for (int r = 0; r < R; ++r) a0[r] = load_a(a[r] + v * V);
#pragma unroll
    for (int r = 0; r < R; ++r) a1[r] = load_a(a[r] + (v + STEP) * V);
    const XVec<TA> x0 = load_x<TA>(x + v * V), x1 = load_x<TA>(x + (v + STEP) * V);
#pragma unroll
    for (int r = 0; r < R; ++r) {
#pragma unroll
      for (int e = 0; e < V; ++e) Tr::fma_(acc[r], a0[r].v[e], x0.v[e], false);
#pragma unroll
      for (int e = 0; e < V; ++e) Tr::fma_(acc[r], a1[r].v[e], x1.v[e], false);
    }
  }
  for (; v < nvec; v += STEP) {
    const XVec<TA> x0 = load_x<TA>(x + v * V);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const AVec<TA> a0 = load_a(a[r] + v * V);
#pragma unroll
      for (int e = 0; e < V; ++e) Tr::fma_(acc[r], a0.v[e], x0.v[e], false);
    }
  }
  if (warp == 0)
    for (size_t jj = nvec * V + lane; jj < n; jj += 32) {
#pragma unroll
      for (int r = 0; r < R; ++r) Tr::fma_(acc[r], a[r][jj], x[jj], false);
    }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    Acc s = acc[r];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = Tr::add(s, shfl_xor_t(s, o));
    if (lane == 0) part[warp][r] = s;
  }
  __syncthreads();
  if (threadIdx.x < R && row0 + threadIdx.x < m) {
    Acc s = part[0][threadIdx.x];
#pragma unroll
    for (int w = 1; w < GS_WARPS; ++w) s = Tr::add(s, part[w][threadIdx.x]);
    y[row0 + threadIdx.x] = s;
  }
}

// -------------------------------------------------------------------------
// op = T / H : y_j = sum_i op(A_ij) x_i
// grid = (column tiles, row chunks of `rows` rows); CTA = 8 warps; lane <-> 16-byte column vector
// -------------------------------------------------------------------------
constexpr int GT_WARPS = 8;
constexpr size_t GT_ROWS = 128;   // rows per chunk while m fits in B2_GRID_Y_MAX chunks; a multiple of it beyond

// TALL: chunks of `rows` rows, a multiple of GT_ROWS (m > B2_GRID_Y_MAX * GT_ROWS); otherwise chunks of GT_ROWS rows
template <typename TA, bool VEC, bool TALL>
__global__ void __launch_bounds__(GT_WARPS * 32)
gemv_t_kernel(const TA* __restrict__ A, size_t lda, size_t m, size_t n,
              const typename ElemTraits<TA>::X* __restrict__ x,
              typename ElemTraits<TA>::X* __restrict__ y,
              typename ElemTraits<TA>::Acc* __restrict__ partials,
              unsigned int* __restrict__ tickets, size_t rows, bool conj) {
  using Tr = ElemTraits<TA>;
  using Acc = typename Tr::Acc;
  constexpr int V = VEC ? Tr::V : 1;
  constexpr int TILE = 32 * V;   // columns per CTA
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t col0 = (size_t)blockIdx.x * TILE + (size_t)lane * V;
  Acc acc[V];
#pragma unroll
  for (int e = 0; e < V; ++e) acc[e] = Tr::zero();
  // rows [r0, r1) of the chunk, r1 - r0 <= GT_ROWS: each lane adds its rows in ascending order
  auto add_rows = [&](const size_t r0, const size_t r1) {
    if (VEC) {
      if (col0 + V <= n) {
        size_t i = r0 + warp;
        // 4 rows in flight per warp
        for (; i + 3 * GT_WARPS < r1; i += 4 * GT_WARPS) {
          AVec<TA> av[4];
          typename Tr::X xv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) av[u] = load_a(A + (i + u * GT_WARPS) * lda + col0);
#pragma unroll
          for (int u = 0; u < 4; ++u) xv[u] = ldg_t(x + i + u * GT_WARPS);
#pragma unroll
          for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int e = 0; e < V; ++e) Tr::fma_(acc[e], av[u].v[e], xv[u], conj);
        }
        for (; i < r1; i += GT_WARPS) {
          AVec<TA> av = load_a(A + i * lda + col0);
          typename Tr::X xv = ldg_t(x + i);
#pragma unroll
          for (int e = 0; e < V; ++e) Tr::fma_(acc[e], av.v[e], xv, conj);
        }
      } else {
        for (size_t i = r0 + warp; i < r1; i += GT_WARPS) {
          typename Tr::X xv = x[i];
#pragma unroll
          for (int e = 0; e < V; ++e)
            if (col0 + e < n) Tr::fma_(acc[e], A[i * lda + col0 + e], xv, conj);
        }
      }
    } else {
      if (col0 < n)
        for (size_t i = r0 + warp; i < r1; i += GT_WARPS) Tr::fma_(acc[0], A[i * lda + col0], x[i], conj);
    }
  };
  if (!TALL) {
    const size_t c0 = (size_t)blockIdx.y * GT_ROWS;
    add_rows(c0, (c0 + GT_ROWS < m) ? c0 + GT_ROWS : m);
  } else {   // the taller chunk in slices of GT_ROWS rows
    const size_t c0 = (size_t)blockIdx.y * rows, c1 = (c0 + rows < m) ? c0 + rows : m;
    for (size_t r0 = c0; r0 < c1; r0 += GT_ROWS) add_rows(r0, (r0 + GT_ROWS < c1) ? r0 + GT_ROWS : c1);
  }
  // fold the 8 warps through shared memory (fixed order)
  __shared__ Acc smem[GT_WARPS][32 * (VEC ? Tr::V : 1)];
  __shared__ bool is_last;
#pragma unroll
  for (int e = 0; e < V; ++e) smem[warp][lane * V + e] = acc[e];
  __syncthreads();
  const int nchunks = gridDim.y;
  for (int c = threadIdx.x; c < TILE; c += GT_WARPS * 32) {
    Acc s = smem[0][c];
#pragma unroll
    for (int w = 1; w < GT_WARPS; ++w) s = Tr::add(s, smem[w][c]);
    const size_t col = (size_t)blockIdx.x * TILE + c;
    if (col < n) {
      if (nchunks == 1) y[col] = s;
      else partials[(size_t)blockIdx.y * n + col] = s;
    }
  }
  if (nchunks == 1) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = atomicAdd(&tickets[blockIdx.x], 1u);
    is_last = (t == (unsigned)nchunks - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    for (int c = threadIdx.x; c < TILE; c += GT_WARPS * 32) {
      const size_t col = (size_t)blockIdx.x * TILE + c;
      if (col < n) {
        Acc s = ldcg_t(&partials[col]);
        for (int k = 1; k < nchunks; ++k) s = Tr::add(s, ldcg_t(&partials[(size_t)k * n + col]));
        y[col] = s;
      }
    }
    if (threadIdx.x == 0) tickets[blockIdx.x] = 0u;
  }
}


// The chunk partials of the transposed gemv only grow (to at least twice their size), and a buffer they outgrow stays
// allocated until b2_ctx_destroy: an address a CUDA graph captured stays valid, and work still in flight on the old
// buffer needs no synchronisation.  Nothing is allocated while the stream is capturing: B2_ERR_WORKSPACE.
int reserve_gemv_partials(b2_ctx* ctx, size_t need, cudaStream_t st) {
  if (need <= ctx->gemv_partials_bytes) return B2_OK;
  cudaStreamCaptureStatus capturing;
  B2_CUDA(cudaStreamIsCapturing(st, &capturing));
  if (capturing != cudaStreamCaptureStatusNone) return B2_ERR_WORKSPACE;
  if (ctx->gemv_partials && ctx->gemv_retired_n == B2_GEMV_RETIRED_MAX) return B2_ERR_WORKSPACE;
  const size_t bytes = need > 2 * ctx->gemv_partials_bytes ? need : 2 * ctx->gemv_partials_bytes;
  float* p = nullptr;
  B2_CUDA(cudaMalloc((void**)&p, bytes));
  if (ctx->gemv_partials) ctx->gemv_retired[ctx->gemv_retired_n++] = ctx->gemv_partials;
  ctx->gemv_partials = p;
  ctx->gemv_partials_bytes = bytes;
  return B2_OK;
}

template <typename TA>
int launch_gemv(b2_ctx* ctx, const void* A, size_t lda, size_t m, size_t n, const void* x,
                void* y, int op, cudaStream_t st) {
  using Tr = ElemTraits<TA>;
  using X = typename Tr::X;
  using Acc = typename Tr::Acc;
  constexpr int V = Tr::V;
  const bool vec = b2_aligned16(A) && ((lda * sizeof(TA)) % 16 == 0);
  if (op == B2_OP_N) {
    if (m == 0) return B2_OK;
    unsigned grid = (unsigned)((m + GN_WARPS - 1) / GN_WARPS);
    if (vec && b2_aligned16(x) && n * sizeof(TA) >= 32768) {
      constexpr int R = 4;
      gemv_n_split_kernel<TA, R><<<(unsigned)((m + R - 1) / R), GS_WARPS * 32, 0, st>>>((const TA*)A, lda, m, n, (const X*)x,
                                                                                        (X*)y);
      B2_LAUNCH_CHECK();
      return B2_OK;
    }
    if (vec && b2_aligned16(x) && n >= (size_t)V)
      gemv_n_kernel<TA, true><<<grid, GN_WARPS * 32, 0, st>>>((const TA*)A, lda, m, n, (const X*)x, (X*)y);
    else
      gemv_n_kernel<TA, false><<<grid, GN_WARPS * 32, 0, st>>>((const TA*)A, lda, m, n, (const X*)x, (X*)y);
    B2_LAUNCH_CHECK();
    return B2_OK;
  }
  if (n == 0) return B2_OK;
  const bool conj = (op == B2_OP_H);
  const size_t tile = 32 * (vec ? V : 1);
  const size_t ntiles = (n + tile - 1) / tile;
  // m >= 1 here.  Chunks of GT_ROWS rows, taller ones once m needs more than B2_GRID_Y_MAX of them
  const size_t rows = GT_ROWS * ((m + GT_ROWS * B2_GRID_Y_MAX - 1) / (GT_ROWS * B2_GRID_Y_MAX));
  const size_t nchunks = (m + rows - 1) / rows;
  // with several chunks the column tiles take tickets (ctx->tickets[64 ..]; slot 0 is the reduction ticket) and
  // are issued in groups of at most that many tiles, one launch per group, each group reusing the tickets and the
  // chunk partials of the previous one (stream order); one chunk needs neither
  const size_t per_launch = nchunks > 1 ? (size_t)(B2_TICKETS - 64) : (size_t)INT_MAX;
  if (nchunks > 1) {
    const size_t group_cols = n < per_launch * tile ? n : per_launch * tile;
    const int rc = reserve_gemv_partials(ctx, nchunks * group_cols * sizeof(Acc), st);
    if (rc) return rc;
  }
  unsigned int* tk = ctx->tickets + 64;
  return b2_launch_groups(ntiles, per_launch, [&](size_t t0, size_t nt) {
    const size_t c0 = t0 * tile, nc = n - c0 < nt * tile ? n - c0 : nt * tile;
    const dim3 grid((unsigned)nt, (unsigned)nchunks);
    const auto kernel = vec ? (rows == GT_ROWS ? gemv_t_kernel<TA, true, false> : gemv_t_kernel<TA, true, true>)
                            : (rows == GT_ROWS ? gemv_t_kernel<TA, false, false> : gemv_t_kernel<TA, false, true>);
    kernel<<<grid, GT_WARPS * 32, 0, st>>>((const TA*)A + c0, lda, m, nc, (const X*)x, (X*)y + c0,
                                           (Acc*)ctx->gemv_partials, tk, rows, conj);
  });
}

}  // namespace

extern "C" int b2_gemv(b2_ctx* ctx, const void* A, size_t lda, size_t m, size_t n, const void* x,
                       void* y, int op, int dtype_a, int dtype_xy, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (op != B2_OP_N && op != B2_OP_T && op != B2_OP_H) return B2_ERR_ARG;
  if (m == 0 && n == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  // empty contraction -> zero output
  const size_t out_len = (op == B2_OP_N) ? m : n, in_len = (op == B2_OP_N) ? n : m;
  if (in_len == 0) {
    if (out_len) B2_CUDA(cudaMemsetAsync(y, 0, out_len * b2_dtype_size(dtype_xy), st));
    return B2_OK;
  }
  if (!A || !x || !y) return B2_ERR_ARG;
  if (lda < n) return B2_ERR_ARG;
  if (dtype_a == B2_BF16) {
    if (dtype_xy != B2_F32) return B2_ERR_DTYPE;
    return launch_gemv<__nv_bfloat16>(ctx, A, lda, m, n, x, y, op, st);
  }
  if (dtype_a != dtype_xy) return B2_ERR_DTYPE;
  return b2_dispatch(dtype_a, [&](auto t) { return launch_gemv<decltype(t)>(ctx, A, lda, m, n, x, y, op, st); });
}
