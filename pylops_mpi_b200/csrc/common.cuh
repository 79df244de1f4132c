// Shared helpers for libb200lops (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <math.h>
#include <stdint.h>
#include <stddef.h>
#include <type_traits>
#include "../../include/b200lops.h"

#define B2_CUDA(call)                                  \
  do {                                                 \
    cudaError_t e__ = (call);                          \
    if (e__ != cudaSuccess) return (int)e__;           \
  } while (0)

#define B2_LAUNCH_CHECK()                              \
  do {                                                 \
    cudaError_t e__ = cudaGetLastError();              \
    if (e__ != cudaSuccess) return (int)e__;           \
  } while (0)

constexpr int B2_GEMV_RETIRED_MAX = 48;   // the gemv scratch doubles as it grows: 48 retired buffers are never reached

struct b2_ctx {
  int device;
  int sm_count;
  // reduction workspace: partial sums + ticket counters (device memory)
  double* red_partials;     // B2_RED_MAX_BLOCKS * B2_RED_MAX_OUT doubles
  unsigned int* tickets;    // B2_TICKETS uints, zero between launches
  float* gemv_partials;     // scratch for transposed gemv (bytes = gemv_partials_bytes); grows, never shrinks
  size_t gemv_partials_bytes;
  float* gemv_retired[B2_GEMV_RETIRED_MAX];  // buffers gemv_partials outgrew, freed by b2_ctx_destroy
  int gemv_retired_n;
  // host-buffer pipeline (b2_first_derivative_host)
  void* pipe_buf[3][2];     // [slot][in/out]
  size_t pipe_bytes;
  cudaStream_t pipe_stream[3];
  cudaEvent_t pipe_ev[3][3];
};

constexpr int B2_RED_MAX_BLOCKS = 2048;
constexpr int B2_RED_MAX_OUT = 16;     // doubles per block (k<=8 complex dots)
constexpr int B2_TICKETS = 4096;

static inline size_t b2_dtype_size(int dt) {
  switch (dt) {
    case B2_F32: return 4;
    case B2_F64: return 8;
    case B2_C64: return 8;
    case B2_C128: return 16;
    case B2_BF16: return 2;
    case B2_I64: return 8;
    default: return 0;
  }
}

static inline bool b2_aligned16(const void* p) { return (((uintptr_t)p) & 15u) == 0; }

// ---- element types and dtype dispatch ----
// A complex element: two R, aligned as R (the float2 / double2 of b2_pair_t are the aligned pair for one 8- / 16-byte
// access).  Complex data can also be handed to a real kernel as 2 n interleaved b2_real_t.
template <typename R>
struct b2_cx { R re, im; };
template <typename R>
using b2_pair_t = typename std::conditional<sizeof(R) == 4, float2, double2>::type;

template <typename T>
struct b2_real { using type = T; };
template <typename R>
struct b2_real<b2_cx<R>> { using type = R; };
template <typename T>
using b2_real_t = typename b2_real<T>::type;
template <typename T>
constexpr bool b2_is_cx_v = false;
template <typename R>
constexpr bool b2_is_cx_v<b2_cx<R>> = true;

template <typename R>
__device__ __forceinline__ b2_cx<R> b2_cx_conj(b2_cx<R> a) { return {a.re, -a.im}; }
template <typename R>
__device__ __forceinline__ b2_cx<R> b2_cx_add(b2_cx<R> a, b2_cx<R> b) { return {a.re + b.re, a.im + b.im}; }
// acc += a x as two explicit fma chains (the products' rounding is fixed: the dense products rely on it)
template <typename R>
__device__ __forceinline__ void b2_cx_fma(b2_cx<R>& acc, b2_cx<R> a, b2_cx<R> x) {
  acc.re = fma(a.re, x.re, fma(-a.im, x.im, acc.re));
  acc.im = fma(a.re, x.im, fma(a.im, x.re, acc.im));
}
// a b as the plain expression, which the compiler may contract (it rounds differently from b2_cx_fma)
template <typename R>
__device__ __forceinline__ b2_cx<R> b2_cx_mul(b2_cx<R> a, b2_cx<R> b) {
  return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}

// f(T()) with T the element type of dtype: float, double, b2_cx<float> or b2_cx<double>; B2_ERR_DTYPE for any other
template <typename F>
int b2_dispatch(int dtype, F f) {
  switch (dtype) {
    case B2_F32: return f(float());
    case B2_F64: return f(double());
    case B2_C64: return f(b2_cx<float>());
    case B2_C128: return f(b2_cx<double>());
    default: return B2_ERR_DTYPE;
  }
}
// the same for the real-only kernels (no complex instantiation is compiled into them)
template <typename F>
int b2_dispatch_real(int dtype, F f) {
  switch (dtype) {
    case B2_F32: return f(float());
    case B2_F64: return f(double());
    default: return B2_ERR_DTYPE;
  }
}

// ---- launch scaffold ----
// launch(first, count) over [0, total) in groups of at most per_launch, where one grid cannot hold them all (gridDim.y
// holds B2_GRID_Y_MAX outer indices, a 1-D grid 2^31 - 1 blocks); stops at the first launch error
constexpr size_t B2_GRID_Y_MAX = 65535;
template <typename F>
int b2_launch_groups(size_t total, size_t per_launch, F launch) {
  for (size_t first = 0; first < total; first += per_launch) {
    launch(first, total - first < per_launch ? total - first : per_launch);
    B2_LAUNCH_CHECK();
  }
  return B2_OK;
}

// a launch of Kernel with more than the default 48 KB of dynamic shared memory has to be allowed first: done once per
// kernel, and again only for a larger size
template <auto Kernel>
int b2_allow_smem(size_t smem) {
  static size_t allowed = 48 * 1024;
  if (smem > allowed) {
    B2_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    allowed = smem;
  }
  return B2_OK;
}

// ---- streaming 16-byte global loads / stores (read-once data: bypass L1) ----
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// coherent variant: safe when the kernel writes the same buffer (in-place ops)
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void stg_stream16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

template <typename T>
struct Vec16;  // 16-byte vector of T
template <>
struct Vec16<float> {
  static constexpr int N = 4;
  float v[4];
};
template <>
struct Vec16<double> {
  static constexpr int N = 2;
  double v[2];
};

// V consecutive elements, aligned to their size so that shared-memory reads of a whole vector compile to one
// LDS.64 / LDS.128 (Vec16 is only element-aligned: the compiler would split it into conflicting scalar reads)
template <typename T, int V>
struct alignas(V * sizeof(T)) VecN { T v[V]; };

template <typename T>
__device__ __forceinline__ Vec16<T> load_vec(const T* p) {
  uint4 r = ldg_stream16(p);
  Vec16<T> o;
  *reinterpret_cast<uint4*>(&o) = r;
  return o;
}
template <typename T>
__device__ __forceinline__ Vec16<T> load_vec_coherent(const T* p) {
  uint4 r = ld_stream16(p);
  Vec16<T> o;
  *reinterpret_cast<uint4*>(&o) = r;
  return o;
}
template <typename T>
__device__ __forceinline__ void store_vec(T* p, const Vec16<T>& v) {
  stg_stream16(p, *reinterpret_cast<const uint4*>(&v));
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- deterministic grid reduction -----------------------------------------------------------------------------------
// The fused reduction kernels (reduce.cu, sparsity.cu, lsqr.cu) run CTAs of B2_RED_THREADS threads on a grid sized by
// b2_red_grid and end in b2_grid_fold.  Their float64 results depend on the grid size and on nothing else, so a call
// repeats its bits; a different grid (or fold order) gives different bits.
constexpr int B2_RED_THREADS = 256;
enum { RED_SUM = 0, RED_MAX = 1, RED_MIN = 2 };

// max / min that return NaN when either operand is NaN, as np.max and np.linalg.norm(x, inf) do (fmax / fmin drop it)
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ double nan_min(double a, double b) { return (a < b || a != a) ? a : b; }

template <int OP>
__device__ __forceinline__ double comb(double a, double b) {
  if (OP == RED_SUM) return a + b;
  if (OP == RED_MAX) return nan_max(a, b);
  return nan_min(a, b);
}
template <int OP>
__device__ __forceinline__ double ident() {
  if (OP == RED_SUM) return 0.0;
  if (OP == RED_MAX) return 0.0;  // all candidates are |x| >= 0
  return INFINITY;
}
template <int OP>
__device__ __forceinline__ double warp_comb(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = comb<OP>(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ceil(items / items_per_cta) CTAs, at least 1 and at most min(8 * SMs, B2_RED_MAX_BLOCKS)
static inline int b2_red_grid(const b2_ctx* ctx, size_t items, size_t items_per_cta) {
  size_t cap = (size_t)ctx->sm_count * 8;
  if (cap > (size_t)B2_RED_MAX_BLOCKS) cap = B2_RED_MAX_BLOCKS;
  const size_t need = (items + items_per_cta - 1) / items_per_cta;
  return (int)(need < 1 ? 1 : (need < cap ? need : cap));
}

struct b2_fold_nothing {
  __device__ void operator()() const {}
};

// Folds acc[0..K) of every thread of the grid into out[0..K) (out may be null); every thread of every CTA calls it,
// as the last statement of the kernel.  A CTA reduces each accumulator with an xor-shuffle tree per warp, then the
// per-warp values in warp 0, and writes its partial to partials[blockIdx.x * K + k].  The last CTA to take the
// ticket folds the partials in CTA order (lane l takes CTAs l, l + 32, ..., then a shuffle tree); the thread that
// writes out then runs last() (a caller's own extra store, made after every CTA has passed its loop) and resets the
// ticket for the next launch.
template <int K, int OP, typename Last = b2_fold_nothing>
__device__ __forceinline__ void b2_grid_fold(const double* acc, double* __restrict__ partials,
                                             unsigned int* __restrict__ ticket, double* __restrict__ out,
                                             Last last = Last()) {
  static_assert(K <= B2_RED_MAX_OUT, "partials hold B2_RED_MAX_OUT doubles per CTA");
  __shared__ double smem[K][B2_RED_THREADS / 32];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const double v = warp_comb<OP>(acc[k]);
    if (lane == 0) smem[k][warp] = v;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double v = warp_comb<OP>(lane < B2_RED_THREADS / 32 ? smem[k][lane] : ident<OP>());
      if (lane == 0) partials[(size_t)blockIdx.x * K + k] = v;
    }
  }
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (warp != 0) return;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double v = ident<OP>();
    for (unsigned int b = lane; b < gridDim.x; b += 32) v = comb<OP>(v, __ldcg(&partials[(size_t)b * K + k]));
    v = warp_comb<OP>(v);
    if (lane == 0 && out) out[k] = v;
  }
  if (lane == 0) {
    last();
    *ticket = 0u;
  }
}
