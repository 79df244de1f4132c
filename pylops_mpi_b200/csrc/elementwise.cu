// Element-wise kernels behind DistributedArray arithmetic
// (reference: pylops_mpi/DistributedArray.py:574-652, 760-837).
// HBM-bound streams: 16-byte vector loads/stores, 4 vectors in flight per
// thread, grid = SMs x 8 persistent CTAs (grid-stride).
#include "common.cuh"

namespace {

constexpr int EW_THREADS = 256;
constexpr int EW_UNROLL = 4;

// ---- real-coefficient linear combination on real data ---------------------
template <typename T, bool HAS_Y>
__global__ void __launch_bounds__(EW_THREADS)
lincomb_vec_kernel(T* __restrict__ out, const T* x, const T* y, double a_scale, double b_scale,
                   const double* __restrict__ a_dev, const double* __restrict__ b_dev,
                   size_t nvec, size_t n) {
  constexpr int V = Vec16<T>::N;
  // a = a_scale * (*a_dev) in double, rounded to T once (the same coefficient axpby_norm2_kernel uses)
  const T a = (T)(a_dev ? a_scale * *a_dev : a_scale), b = (T)(b_dev ? b_scale * *b_dev : b_scale);
  const size_t stride = (size_t)gridDim.x * EW_THREADS;
  size_t i = (size_t)blockIdx.x * EW_THREADS + threadIdx.x;
  for (; i + (EW_UNROLL - 1) * stride < nvec; i += EW_UNROLL * stride) {
    Vec16<T> vx[EW_UNROLL], vy[EW_UNROLL];
#pragma unroll
    for (int u = 0; u < EW_UNROLL; ++u) vx[u] = load_vec_coherent(x + (i + u * stride) * V);
    if (HAS_Y) {
#pragma unroll
      for (int u = 0; u < EW_UNROLL; ++u) vy[u] = load_vec_coherent(y + (i + u * stride) * V);
    }
#pragma unroll
    for (int u = 0; u < EW_UNROLL; ++u) {
      Vec16<T> o;
#pragma unroll
      for (int k = 0; k < V; ++k) o.v[k] = HAS_Y ? a * vx[u].v[k] + b * vy[u].v[k] : a * vx[u].v[k];
      store_vec(out + (i + u * stride) * V, o);
    }
  }
  for (; i < nvec; i += stride) {
    Vec16<T> vx = load_vec_coherent(x + i * V), o;
    if (HAS_Y) {
      Vec16<T> vy = load_vec_coherent(y + i * V);
#pragma unroll
      for (int k = 0; k < V; ++k) o.v[k] = a * vx.v[k] + b * vy.v[k];
    } else {
#pragma unroll
      for (int k = 0; k < V; ++k) o.v[k] = a * vx.v[k];
    }
    store_vec(out + i * V, o);
  }
  // scalar tail (n % V elements)
  if (blockIdx.x == 0) {
    size_t t = nvec * V + threadIdx.x;
    if (t < n) out[t] = HAS_Y ? a * x[t] + b * y[t] : a * x[t];
  }
}

template <typename T, bool HAS_Y>
__global__ void __launch_bounds__(EW_THREADS)
lincomb_scalar_kernel(T* out, const T* x, const T* y, double a_scale, double b_scale, const double* a_dev,
                      const double* b_dev, size_t n) {
  const T a = (T)(a_dev ? a_scale * *a_dev : a_scale), b = (T)(b_dev ? b_scale * *b_dev : b_scale);
  const size_t stride = (size_t)gridDim.x * EW_THREADS;
  for (size_t i = (size_t)blockIdx.x * EW_THREADS + threadIdx.x; i < n; i += stride)
    out[i] = HAS_Y ? a * x[i] + b * y[i] : a * x[i];
}

// ---- complex path (complex coefficients and/or conj) ----------------------
template <typename R, bool HAS_Y, bool CONJ>
__global__ void __launch_bounds__(EW_THREADS)
lincomb_cx_kernel(b2_cx<R>* out, const b2_cx<R>* x, const b2_cx<R>* y, b2_cx<R> a, b2_cx<R> b, size_t n) {
  const size_t stride = (size_t)gridDim.x * EW_THREADS;
  for (size_t i = (size_t)blockIdx.x * EW_THREADS + threadIdx.x; i < n; i += stride) {
    b2_cx<R> xv = x[i];
    if (CONJ) xv.im = -xv.im;
    b2_cx<R> o = b2_cx_mul(a, xv);
    if (HAS_Y) {
      b2_cx<R> t = b2_cx_mul(b, y[i]);
      o.re += t.re;
      o.im += t.im;
    }
    out[i] = o;
  }
}

template <typename T>
__global__ void __launch_bounds__(EW_THREADS)
mul_real_kernel(T* out, const T* x, const T* y, size_t n) {
  const size_t stride = (size_t)gridDim.x * EW_THREADS;
  for (size_t i = (size_t)blockIdx.x * EW_THREADS + threadIdx.x; i < n; i += stride)
    out[i] = x[i] * y[i];
}
template <typename R, bool CONJ>
__global__ void __launch_bounds__(EW_THREADS)
mul_cx_kernel(b2_cx<R>* out, const b2_cx<R>* x, const b2_cx<R>* y, size_t n) {
  const size_t stride = (size_t)gridDim.x * EW_THREADS;
  for (size_t i = (size_t)blockIdx.x * EW_THREADS + threadIdx.x; i < n; i += stride) {
    b2_cx<R> xv = x[i];
    if (CONJ) xv.im = -xv.im;
    out[i] = b2_cx_mul(xv, y[i]);
  }
}

template <typename T>
__global__ void __launch_bounds__(EW_THREADS) fill_kernel(T* out, T v, size_t n) {
  const size_t stride = (size_t)gridDim.x * EW_THREADS;
  for (size_t i = (size_t)blockIdx.x * EW_THREADS + threadIdx.x; i < n; i += stride) out[i] = v;
}

inline int ew_grid(const b2_ctx* ctx, size_t work_items) {
  size_t need = (work_items + EW_THREADS - 1) / EW_THREADS;
  size_t cap = (size_t)ctx->sm_count * 8;
  if (need < 1) need = 1;
  return (int)(need < cap ? need : cap);
}

template <typename T>
int lincomb_real(b2_ctx* ctx, T* out, const T* x, const T* y, double a, double b,
                 const double* a_dev, const double* b_dev, size_t n, cudaStream_t st) {
  if (n == 0) return B2_OK;
  constexpr int V = Vec16<T>::N;
  const bool aligned = b2_aligned16(out) && b2_aligned16(x) && (!y || b2_aligned16(y));
  if (aligned && n >= (size_t)V) {
    size_t nvec = n / V;
    int grid = ew_grid(ctx, (nvec + EW_UNROLL - 1) / EW_UNROLL);
    if (y)
      lincomb_vec_kernel<T, true><<<grid, EW_THREADS, 0, st>>>(out, x, y, a, b, a_dev, b_dev, nvec, n);
    else
      lincomb_vec_kernel<T, false><<<grid, EW_THREADS, 0, st>>>(out, x, y, a, b, a_dev, b_dev, nvec, n);
  } else {
    int grid = ew_grid(ctx, n);
    if (y)
      lincomb_scalar_kernel<T, true><<<grid, EW_THREADS, 0, st>>>(out, x, y, a, b, a_dev, b_dev, n);
    else
      lincomb_scalar_kernel<T, false><<<grid, EW_THREADS, 0, st>>>(out, x, y, a, b, a_dev, b_dev, n);
  }
  B2_LAUNCH_CHECK();
  return B2_OK;
}

template <typename R>
int lincomb_cx(b2_ctx* ctx, void* out, const void* x, const void* y, const double a[2],
               const double b[2], size_t n, int conj_x, cudaStream_t st) {
  if (n == 0) return B2_OK;
  int grid = ew_grid(ctx, n);
  b2_cx<R> ca{(R)a[0], (R)a[1]}, cb{(R)(b ? b[0] : 0.0), (R)(b ? b[1] : 0.0)};
  auto o = (b2_cx<R>*)out;
  auto xx = (const b2_cx<R>*)x;
  auto yy = (const b2_cx<R>*)y;
  if (y) {
    if (conj_x) lincomb_cx_kernel<R, true, true><<<grid, EW_THREADS, 0, st>>>(o, xx, yy, ca, cb, n);
    else lincomb_cx_kernel<R, true, false><<<grid, EW_THREADS, 0, st>>>(o, xx, yy, ca, cb, n);
  } else {
    if (conj_x) lincomb_cx_kernel<R, false, true><<<grid, EW_THREADS, 0, st>>>(o, xx, yy, ca, cb, n);
    else lincomb_cx_kernel<R, false, false><<<grid, EW_THREADS, 0, st>>>(o, xx, yy, ca, cb, n);
  }
  B2_LAUNCH_CHECK();
  return B2_OK;
}

}  // namespace

extern "C" int b2_lincomb(b2_ctx* ctx, void* out, const double a[2], const void* x,
                          const double b[2], const void* y, size_t n, int dtype, int conj_x,
                          void* stream) {
  if (!ctx || !out || !x || !a) return B2_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const double bz[2] = {0.0, 0.0};
  if (!b) b = bz;
  const bool real_coef = (a[1] == 0.0) && (!y || b[1] == 0.0);
  return b2_dispatch(dtype, [&](auto t) {
    using T = decltype(t);
    using R = b2_real_t<T>;
    // complex data with real coefficients and no conj: the real kernel on 2 n reals
    if constexpr (b2_is_cx_v<T>) {
      if (!real_coef || conj_x) return lincomb_cx<R>(ctx, out, x, y, a, b, n, conj_x, st);
    }
    return lincomb_real<R>(ctx, (R*)out, (const R*)x, (const R*)y, a[0], b[0], nullptr, nullptr,
                           b2_is_cx_v<T> ? 2 * n : n, st);
  });
}

extern "C" int b2_lincomb_dev(b2_ctx* ctx, void* out, const double* a_dev, double a_scale,
                              const void* x, const double* b_dev, double b_scale, const void* y,
                              size_t n, int dtype, void* stream) {
  if (!ctx || !out || !x) return B2_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  // real coefficients: complex data runs as 2 n reals
  return b2_dispatch(dtype, [&](auto t) {
    using R = b2_real_t<decltype(t)>;
    return lincomb_real<R>(ctx, (R*)out, (const R*)x, (const R*)y, a_scale, b_scale, a_dev, b_dev,
                           b2_is_cx_v<decltype(t)> ? 2 * n : n, st);
  });
}

extern "C" int b2_mul(b2_ctx* ctx, void* out, const void* x, const void* y, size_t n, int dtype,
                      int conj_x, void* stream) {
  if (!ctx || !out || !x || !y) return B2_ERR_ARG;
  if (n == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int grid = ew_grid(ctx, n);
  return b2_dispatch(dtype, [&](auto t) -> int {
    using T = decltype(t);
    if constexpr (b2_is_cx_v<T>) {
      using R = b2_real_t<T>;
      if (conj_x) mul_cx_kernel<R, true><<<grid, EW_THREADS, 0, st>>>((T*)out, (const T*)x, (const T*)y, n);
      else mul_cx_kernel<R, false><<<grid, EW_THREADS, 0, st>>>((T*)out, (const T*)x, (const T*)y, n);
    } else {
      mul_real_kernel<T><<<grid, EW_THREADS, 0, st>>>((T*)out, (const T*)x, (const T*)y, n);
    }
    B2_LAUNCH_CHECK();
    return B2_OK;
  });
}

extern "C" int b2_fill(b2_ctx* ctx, void* out, const double v[2], size_t n, int dtype,
                       void* stream) {
  if (!ctx || !out || !v) return B2_ERR_ARG;
  if (n == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int grid = ew_grid(ctx, n);
  return b2_dispatch(dtype, [&](auto t) -> int {
    using T = decltype(t);
    if constexpr (b2_is_cx_v<T>) {   // one 8- / 16-byte store per complex element
      using P = b2_pair_t<b2_real_t<T>>;
      fill_kernel<P><<<grid, EW_THREADS, 0, st>>>((P*)out, P{(b2_real_t<T>)v[0], (b2_real_t<T>)v[1]}, n);
    } else {
      fill_kernel<T><<<grid, EW_THREADS, 0, st>>>((T*)out, (T)v[0], n);
    }
    B2_LAUNCH_CHECK();
    return B2_OK;
  });
}


// ---- stationary-A MPIMatrixMult helpers (round 2) -------------------------------------------------------------
// (1) float32 tile -> bfloat16, written to up to 8 destinations (local or IPC-mapped peer buffers): the all-gather of
//     the X / Y panels of MatrixMult.py:663-670, 742-763 with the fp32 -> bf16 cast fused in (one read of the tile).
// (2) out = sum over slots of the partial tiles the peers' GEMM epilogues stored here, in slot order (deterministic).
namespace {
struct CastDst {
  __nv_bfloat16* p[8];
  int n;
};
__global__ void __launch_bounds__(256)
cast_multi_kernel(const float* __restrict__ src, size_t ld_src, size_t rows, size_t cols, CastDst dst, size_t ld_dst, int vec) {
  if (vec) {
    const size_t cv = cols / 8, total = rows * cv;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
      const size_t r = e / cv, c = (e % cv) * 8;
      const float4 a = *reinterpret_cast<const float4*>(src + r * ld_src + c);
      const float4 b = *reinterpret_cast<const float4*>(src + r * ld_src + c + 4);
      __nv_bfloat162 h0 = __floats2bfloat162_rn(a.x, a.y), h1 = __floats2bfloat162_rn(a.z, a.w);
      __nv_bfloat162 h2 = __floats2bfloat162_rn(b.x, b.y), h3 = __floats2bfloat162_rn(b.z, b.w);
      uint4 o;
      o.x = *reinterpret_cast<uint32_t*>(&h0); o.y = *reinterpret_cast<uint32_t*>(&h1);
      o.z = *reinterpret_cast<uint32_t*>(&h2); o.w = *reinterpret_cast<uint32_t*>(&h3);
      for (int d = 0; d < dst.n; ++d) *reinterpret_cast<uint4*>(dst.p[d] + r * ld_dst + c) = o;
    }
  } else {
    const size_t total = rows * cols;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
      const size_t r = e / cols, c = e % cols;
      const __nv_bfloat16 h = __float2bfloat16_rn(src[r * ld_src + c]);
      for (int d = 0; d < dst.n; ++d) dst.p[d][r * ld_dst + c] = h;
    }
  }
}
__global__ void __launch_bounds__(256)
sum_slots_kernel(const float* __restrict__ slots, size_t slot_stride, int nslots, size_t ld_in, float* __restrict__ out,
                 size_t rows, size_t cols, int vec) {
  if (vec) {
    const size_t cv = cols / 4, total = rows * cv;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
      const size_t r = e / cv, c = (e % cv) * 4;
      float4 acc = *reinterpret_cast<const float4*>(slots + r * ld_in + c);
      for (int s = 1; s < nslots; ++s) {
        const float4 v = *reinterpret_cast<const float4*>(slots + (size_t)s * slot_stride + r * ld_in + c);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      *reinterpret_cast<float4*>(out + r * cols + c) = acc;
    }
  } else {
    const size_t total = rows * cols;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
      const size_t r = e / cols, c = e % cols;
      float acc = slots[r * ld_in + c];
      for (int s = 1; s < nslots; ++s) acc += slots[(size_t)s * slot_stride + r * ld_in + c];
      out[r * cols + c] = acc;
    }
  }
}
}  // namespace

extern "C" int b2_cast_bf16_multi(b2_ctx* ctx, const float* src, size_t ld_src, size_t rows, size_t cols,
                                  void* const* dsts_host, int ndst, size_t ld_dst, void* stream) {
  if (!ctx || ndst < 1 || ndst > 8 || !dsts_host) return B2_ERR_ARG;
  if (rows == 0 || cols == 0) return B2_OK;
  if (!src) return B2_ERR_ARG;
  CastDst d;
  d.n = ndst;
  int vec = (cols % 8 == 0) && (ld_src % 4 == 0) && (ld_dst % 8 == 0) && b2_aligned16(src);
  for (int i = 0; i < 8; ++i) {
    d.p[i] = i < ndst ? (__nv_bfloat16*)dsts_host[i] : nullptr;
    if (i < ndst && !dsts_host[i]) return B2_ERR_ARG;
    if (i < ndst && !b2_aligned16(dsts_host[i])) vec = 0;
  }
  const size_t work = vec ? rows * (cols / 8) : rows * cols;
  size_t blocks = (work + 255) / 256;
  const size_t cap = (size_t)ctx->sm_count * 16;
  if (blocks > cap) blocks = cap;
  cast_multi_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, ld_src, rows, cols, d, ld_dst, vec);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

extern "C" int b2_sum_slots(b2_ctx* ctx, const float* slots, size_t slot_stride, int nslots, size_t ld_in, float* out,
                            size_t rows, size_t cols, void* stream) {
  if (!ctx || nslots < 1) return B2_ERR_ARG;
  if (rows == 0 || cols == 0) return B2_OK;
  if (!slots || !out) return B2_ERR_ARG;
  const int vec = (cols % 4 == 0) && (ld_in % 4 == 0) && (slot_stride % 4 == 0) && b2_aligned16(slots) && b2_aligned16(out);
  const size_t work = vec ? rows * (cols / 4) : rows * cols;
  size_t blocks = (work + 255) / 256;
  const size_t cap = (size_t)ctx->sm_count * 16;
  if (blocks > cap) blocks = cap;
  sum_slots_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(slots, slot_stride, nslots, ld_in, out, rows, cols, vec);
  B2_LAUNCH_CHECK();
  return B2_OK;
}
