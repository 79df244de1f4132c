// Generic (f32 / f64 / c64 / c128) dense tile product on the SIMT pipes:
//   C[b] (+)= op(A[b]) B[b],  A[b] is m x k (op=N) or k x m (op=T/H), B[b] k x n, C[b] m x n,
// all row-major, optional batch strides.  Serves
//   * the multi-column tile product of MPIMatrixMult for the dtypes the tensor
//     cores do not cover (pylops_mpi/basicoperators/MatrixMult.py:366-370, 409-413,
//     663-670, 742-763; parity cases of tests/test_matrixmult.py), and
//   * the per-slice product of MPIFredholm1 (signalprocessing/Fredholm1.py:119-129,
//     147-167), one slice per blockIdx.z.
// 64x64 CTA tile, 16-deep K slices through shared memory, 4x4 register tile per
// thread.  The bf16 tensor-core path lives in gemm_tc.cu.
#include <string.h>
#include "common.cuh"

namespace {

template <typename T> struct Num {   // float / double
  __device__ static __forceinline__ T zero() { return T(0); }
  __device__ static __forceinline__ void fma_(T& c, T a, T b) { c = fma(a, b, c); }
  __device__ static __forceinline__ T conj(T a) { return a; }
  __device__ static __forceinline__ T add(T a, T b) { return a + b; }
};
template <typename R> struct Num<b2_cx<R>> {
  using C = b2_cx<R>;
  __device__ static __forceinline__ C zero() { return {R(0), R(0)}; }
  __device__ static __forceinline__ void fma_(C& c, C a, C b) { b2_cx_fma(c, a, b); }
  __device__ static __forceinline__ C conj(C a) { return b2_cx_conj(a); }
  __device__ static __forceinline__ C add(C a, C b) { return b2_cx_add(a, b); }
};

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;

// extra destinations of the SAME logical output buffer in peer GPUs' memory (IPC-mapped, NVLink):
// the epilogue stores every result element locally and to each peer -> the all-gather of
// MPIFredholm1 (Fredholm1.py:131-132) happens inside the product kernel, tile by tile.
struct PeerDst {
  void* p[8];
  int n;
};

template <typename T, bool TRANS_A, bool FUSED = false>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const T* __restrict__ A, size_t lda, size_t sA, const T* __restrict__ B,
                 size_t ldb, size_t sB, T* __restrict__ C, size_t ldc, size_t sC, size_t m,
                 size_t n, size_t k, bool conj_a, bool accumulate, PeerDst peers = PeerDst{}) {
  using N_ = Num<T>;
  __shared__ T As[BK][BM + 1];
  __shared__ T Bs[BK][BN + 1];
  A += (size_t)blockIdx.z * sA;
  B += (size_t)blockIdx.z * sB;
  C += (size_t)blockIdx.z * sC;
  const size_t m0 = (size_t)blockIdx.y * BM, n0 = (size_t)blockIdx.x * BN;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  T acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = N_::zero();

  for (size_t k0 = 0; k0 < k; k0 += BK) {
    // A tile -> As[kk][i]
    for (int e = threadIdx.x; e < BM * BK; e += 256) {
      int i, kk;
      if (TRANS_A) { i = e % BM; kk = e / BM; }   // contiguous along m
      else { kk = e % BK; i = e / BK; }            // contiguous along k
      const size_t gi = m0 + i, gk = k0 + kk;
      T v = N_::zero();
      if (gi < m && gk < k) {
        v = TRANS_A ? A[gk * lda + gi] : A[gi * lda + gk];
        if (conj_a) v = N_::conj(v);
      }
      As[kk][i] = v;
    }
    for (int e = threadIdx.x; e < BN * BK; e += 256) {
      const int j = e % BN, kk = e / BN;
      const size_t gj = n0 + j, gk = k0 + kk;
      Bs[kk][j] = (gj < n && gk < k) ? B[gk * ldb + gj] : N_::zero();
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      T a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) N_::fma_(acc[i][j], a[i], b[j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const size_t gi = m0 + ty * TM + i;
    if (gi >= m) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const size_t gj = n0 + tx + 16 * j;
      if (gj >= n) continue;
      T* c = C + gi * ldc + gj;
      const T v = accumulate ? N_::add(*c, acc[i][j]) : acc[i][j];
      *c = v;
      if (FUSED) {
        const size_t off = (size_t)blockIdx.z * sC + gi * ldc + gj;
        for (int d = 0; d < peers.n; ++d) reinterpret_cast<T*>(peers.p[d])[off] = v;   // P2P store over NVLink
      }
    }
  }
}

// FUSED: the epilogue also stores to the peers (b2_batched_gemm_allgather).  That entry point does not check the grid
// here: an empty or too tall grid is left to the launch, which returns CUDA's error code.  Otherwise more than
// B2_GRID_Y_MAX row tiles are issued in groups of output rows, one launch each: a group starts at row r0 of C and of
// op(A), i.e. row r0 of A for op N and column r0 for op T / H
template <typename T, bool FUSED = false>
int launch_gemm(const void* A, size_t lda, size_t sA, const void* B, size_t ldb, size_t sB,
                void* C, size_t ldc, size_t sC, size_t m, size_t n, size_t k, size_t batch,
                int op_a, bool accumulate, cudaStream_t st, const PeerDst& peers = PeerDst{}) {
  const bool conj = (op_a == B2_OP_H);
  auto launch = [&](size_t r0, size_t rows) {
    const dim3 grid((unsigned)((n + BN - 1) / BN), (unsigned)((rows + BM - 1) / BM), (unsigned)batch);
    T* c = (T*)C + r0 * ldc;
    if (op_a == B2_OP_N)
      gemm_simt_kernel<T, false, FUSED><<<grid, 256, 0, st>>>((const T*)A + r0 * lda, lda, sA, (const T*)B, ldb, sB, c, ldc, sC, rows, n, k, false, accumulate, peers);
    else
      gemm_simt_kernel<T, true, FUSED><<<grid, 256, 0, st>>>((const T*)A + r0, lda, sA, (const T*)B, ldb, sB, c, ldc, sC, rows, n, k, conj, accumulate, peers);
  };
  if (FUSED) {
    launch(0, m);
    B2_LAUNCH_CHECK();
    return B2_OK;
  }
  if (m == 0 || n == 0 || batch == 0) return B2_OK;
  if (batch > 65535) return B2_ERR_ARG;
  return b2_launch_groups(m, B2_GRID_Y_MAX * BM, launch);
}

int dispatch(const void* A, size_t lda, size_t sA, const void* B, size_t ldb, size_t sB, void* C,
             size_t ldc, size_t sC, size_t m, size_t n, size_t k, size_t batch, int op_a,
             bool accumulate, int dtype, cudaStream_t st) {
  return b2_dispatch(dtype, [&](auto t) {
    return launch_gemm<decltype(t)>(A, lda, sA, B, ldb, sB, C, ldc, sC, m, n, k, batch, op_a, accumulate, st);
  });
}

}  // namespace

// y[s] = op(G[s]) x[s] written to the local output AND to the same offsets of `npeers` peer buffers
// (fused product + all-gather over NVLink peer memory).  peers_host[d] must already point at the
// position in peer d's buffer that corresponds to y.
extern "C" int b2_batched_gemm_allgather(b2_ctx* ctx, const void* G, const void* x, void* y,
                                         void* const* peers_host, int npeers, size_t nsl, size_t nx, size_t ny,
                                         size_t nz, int adjoint, int dtype, void* stream) {
  if (!ctx || npeers < 0 || npeers > 8) return B2_ERR_ARG;
  if (nsl == 0) return B2_OK;
  if (!G || !x || !y || (npeers && !peers_host)) return B2_ERR_ARG;
  if (nsl > 65535) return B2_ERR_ARG;
  const size_t m = adjoint ? ny : nx, k = adjoint ? nx : ny;
  PeerDst pd;
  pd.n = npeers;
  for (int d = 0; d < 8; ++d) pd.p[d] = d < npeers ? peers_host[d] : nullptr;
  return b2_dispatch(dtype, [&](auto t) {
    return launch_gemm<decltype(t), true>(G, ny, nx * ny, x, nz, k * nz, y, nz, m * nz, m, nz, k, nsl,
                                          adjoint ? B2_OP_H : B2_OP_N, false, (cudaStream_t)stream, pd);
  });
}

// symmetric (peer-mappable) buffers: plain cudaMalloc + CUDA IPC handles exchanged by the caller
extern "C" int b2_symm_alloc(size_t bytes, void** out) {
  if (!out) return B2_ERR_ARG;
  B2_CUDA(cudaMalloc(out, bytes));
  return B2_OK;
}
extern "C" int b2_symm_free(void* p) {
  if (p) B2_CUDA(cudaFree(p));
  return B2_OK;
}
extern "C" int b2_ipc_get_handle(void* p, void* handle64_host) {
  if (!p || !handle64_host) return B2_ERR_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaIpcMemHandle_t h;
  B2_CUDA(cudaIpcGetMemHandle(&h, p));
  memcpy(handle64_host, &h, sizeof h);
  return B2_OK;
}
extern "C" int b2_ipc_open_handle(const void* handle64_host, void** out) {
  if (!handle64_host || !out) return B2_ERR_ARG;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64_host, sizeof h);
  B2_CUDA(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
  return B2_OK;
}
extern "C" int b2_ipc_close_handle(void* p) {
  if (p) B2_CUDA(cudaIpcCloseMemHandle(p));
  return B2_OK;
}

extern "C" int b2_gemm(b2_ctx* ctx, const void* A, size_t lda, const void* B, size_t ldb, void* C,
                       size_t ldc, size_t m, size_t n, size_t k, int op_a, int accumulate,
                       int dtype, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (op_a != B2_OP_N && op_a != B2_OP_T && op_a != B2_OP_H) return B2_ERR_ARG;
  if (m && n && (!C)) return B2_ERR_ARG;
  if (m && n && k && (!A || !B)) return B2_ERR_ARG;
  return dispatch(A, lda, 0, B, ldb, 0, C, ldc, 0, m, n, k, 1, op_a, accumulate != 0, dtype,
                  (cudaStream_t)stream);
}

extern "C" int b2_batched_gemm(b2_ctx* ctx, const void* G, const void* x, void* y, size_t nsl,
                               size_t nx, size_t ny, size_t nz, int adjoint, int dtype,
                               void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (nsl == 0) return B2_OK;
  if (!G || !x || !y) return B2_ERR_ARG;
  // forward: y[s] (nx x nz) = G[s] (nx x ny) x[s] (ny x nz)
  // adjoint: y[s] (ny x nz) = G[s]^H (ny x nx) x[s] (nx x nz)
  const size_t m = adjoint ? ny : nx, k = adjoint ? nx : ny;
  size_t done = 0;
  while (done < nsl) {   // blockIdx.z limit
    size_t b = nsl - done < 65535 ? nsl - done : 65535;
    const size_t es = b2_dtype_size(dtype);
    int rc = dispatch((const char*)G + done * nx * ny * es, ny, nx * ny,
                      (const char*)x + done * k * nz * es, nz, k * nz,
                      (char*)y + done * m * nz * es, nz, m * nz, m, nz, k, b,
                      adjoint ? B2_OP_H : B2_OP_N, false, dtype, (cudaStream_t)stream);
    if (rc) return rc;
    done += b;
  }
  return B2_OK;
}
