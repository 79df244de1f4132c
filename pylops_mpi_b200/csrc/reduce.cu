// Local (per-rank) reductions behind DistributedArray.dot / norm
// (reference: pylops_mpi/DistributedArray.py:654-686, 688-758).
//
// One launch per reduction: every CTA streams its grid-stride share with
// 16-byte loads, accumulates in float64 registers, and b2_grid_fold (common.cuh)
// folds the per-CTA partials in CTA order, so the result is deterministic for a given n.
// HBM-bound: algorithmic bytes = n*sizeof(T) per operand.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int RED_THREADS = B2_RED_THREADS;
constexpr int RED_UNROLL = 4;

// ---- functors --------------------------------------------------------------
// real(acc, x, y) consumes one real element; cx(acc, xr, xi, yr, yi) one complex.
template <bool CONJ>
struct DotF {
  static constexpr int NOUT_REAL = 1, NOUT_CX = 2, MODE = RED_SUM;
  static constexpr bool HAS_Y = true;
  double p;
  template <typename T>
  __device__ __forceinline__ void real(double* acc, T x, T y) const {
    acc[0] = fma((double)x, (double)y, acc[0]);
  }
  template <typename T>
  __device__ __forceinline__ void cx(double* acc, T xr, T xi, T yr, T yi) const {
    double a = xr, b = CONJ ? -(double)xi : (double)xi, c = yr, d = yi;
    acc[0] += a * c - b * d;
    acc[1] += a * d + b * c;
  }
};
struct SumSqF {
  static constexpr int NOUT_REAL = 1, NOUT_CX = 1, MODE = RED_SUM;
  static constexpr bool HAS_Y = false;
  double p;
  template <typename T>
  __device__ __forceinline__ void real(double* acc, T x, T) const {
    acc[0] = fma((double)x, (double)x, acc[0]);
  }
  template <typename T>
  __device__ __forceinline__ void cx(double* acc, T xr, T xi, T, T) const {
    acc[0] += (double)xr * (double)xr + (double)xi * (double)xi;
  }
};
struct SumAbsF {
  static constexpr int NOUT_REAL = 1, NOUT_CX = 1, MODE = RED_SUM;
  static constexpr bool HAS_Y = false;
  double p;
  template <typename T>
  __device__ __forceinline__ void real(double* acc, T x, T) const { acc[0] += fabs((double)x); }
  template <typename T>
  __device__ __forceinline__ void cx(double* acc, T xr, T xi, T, T) const {
    acc[0] += hypot((double)xr, (double)xi);
  }
};
struct CountNzF {
  static constexpr int NOUT_REAL = 1, NOUT_CX = 1, MODE = RED_SUM;
  static constexpr bool HAS_Y = false;
  double p;
  template <typename T>
  __device__ __forceinline__ void real(double* acc, T x, T) const { acc[0] += (x != (T)0) ? 1.0 : 0.0; }
  template <typename T>
  __device__ __forceinline__ void cx(double* acc, T xr, T xi, T, T) const {
    acc[0] += (xr != (T)0 || xi != (T)0) ? 1.0 : 0.0;
  }
};
template <int M>
struct ExtAbsF {
  static constexpr int NOUT_REAL = 1, NOUT_CX = 1, MODE = M;
  static constexpr bool HAS_Y = false;
  double p;
  template <typename T>
  __device__ __forceinline__ void real(double* acc, T x, T) const { acc[0] = comb<M>(acc[0], fabs((double)x)); }
  template <typename T>
  __device__ __forceinline__ void cx(double* acc, T xr, T xi, T, T) const {
    acc[0] = comb<M>(acc[0], hypot((double)xr, (double)xi));
  }
};
struct SumPowF {
  static constexpr int NOUT_REAL = 1, NOUT_CX = 1, MODE = RED_SUM;
  static constexpr bool HAS_Y = false;
  double p;
  template <typename T>
  __device__ __forceinline__ void real(double* acc, T x, T) const { acc[0] += pow(fabs((double)x), p); }
  template <typename T>
  __device__ __forceinline__ void cx(double* acc, T xr, T xi, T, T) const {
    acc[0] += pow(hypot((double)xr, (double)xi), p);
  }
};

template <typename T, bool CX, typename F>
__device__ __forceinline__ void consume_vec(const F& f, double* acc, const Vec16<T>& vx,
                                            const Vec16<T>& vy) {
  constexpr int V = Vec16<T>::N;
  if (!CX) {
#pragma unroll
    for (int k = 0; k < V; ++k) f.real(acc, vx.v[k], vy.v[k]);
  } else {
#pragma unroll
    for (int k = 0; k < V; k += 2) f.cx(acc, vx.v[k], vx.v[k + 1], vy.v[k], vy.v[k + 1]);
  }
}

// n_real = number of T scalars (2 per complex element).  VEC path requires 16B alignment.
template <typename T, bool CX, bool VEC, typename F>
__global__ void __launch_bounds__(RED_THREADS)
reduce_kernel(F f, const T* __restrict__ x, const T* __restrict__ y, size_t n_real,
              double* __restrict__ partials, unsigned int* __restrict__ ticket,
              double* __restrict__ out) {
  constexpr int NOUT = CX ? F::NOUT_CX : F::NOUT_REAL;
  constexpr int MODE = F::MODE;
  constexpr int V = Vec16<T>::N;
  double acc[NOUT];
#pragma unroll
  for (int k = 0; k < NOUT; ++k) acc[k] = ident<MODE>();

  const size_t stride = (size_t)gridDim.x * RED_THREADS;
  size_t i = (size_t)blockIdx.x * RED_THREADS + threadIdx.x;
  if (VEC) {
    const size_t nvec = n_real / V;
    for (; i + (RED_UNROLL - 1) * stride < nvec; i += RED_UNROLL * stride) {
      Vec16<T> vx[RED_UNROLL], vy[RED_UNROLL];
#pragma unroll
      for (int u = 0; u < RED_UNROLL; ++u) vx[u] = load_vec(x + (i + u * stride) * V);
      if (F::HAS_Y) {
#pragma unroll
        for (int u = 0; u < RED_UNROLL; ++u) vy[u] = load_vec(y + (i + u * stride) * V);
      }
#pragma unroll
      for (int u = 0; u < RED_UNROLL; ++u) consume_vec<T, CX>(f, acc, vx[u], F::HAS_Y ? vy[u] : vx[u]);
    }
    for (; i < nvec; i += stride) {
      Vec16<T> vx = load_vec(x + i * V);
      Vec16<T> vy = vx;
      if (F::HAS_Y) vy = load_vec(y + i * V);
      consume_vec<T, CX>(f, acc, vx, vy);
    }
    // tail scalars (only possible for real data; complex pairs never split a vector
    // except T=float with an odd complex count -> one trailing pair)
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      size_t t = nvec * V;
      if (!CX) {
        for (; t < n_real; ++t) f.real(acc, x[t], F::HAS_Y ? y[t] : x[t]);
      } else {
        for (; t + 1 < n_real; t += 2)
          f.cx(acc, x[t], x[t + 1], F::HAS_Y ? y[t] : x[t], F::HAS_Y ? y[t + 1] : x[t + 1]);
      }
    }
  } else {
    if (!CX) {
      for (; i < n_real; i += stride) f.real(acc, x[i], F::HAS_Y ? y[i] : x[i]);
    } else {
      const size_t nc = n_real / 2;
      for (; i < nc; i += stride)
        f.cx(acc, x[2 * i], x[2 * i + 1], F::HAS_Y ? y[2 * i] : x[2 * i],
             F::HAS_Y ? y[2 * i + 1] : x[2 * i + 1]);
    }
  }
  b2_grid_fold<NOUT, MODE>(acc, partials, ticket, out);
}

// the grid of reduce_kernel, dot_multi_kernel and axpby_norm2_kernel: 1024 items (vectors or scalars) per CTA
inline int red_grid(const b2_ctx* ctx, size_t n_items) { return b2_red_grid(ctx, n_items, RED_THREADS * RED_UNROLL); }

template <typename T, bool CX, typename F>
int launch_reduce(b2_ctx* ctx, F f, const void* x, const void* y, size_t n_real, double* out,
                  cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  const bool vec = b2_aligned16(x) && (!F::HAS_Y || b2_aligned16(y)) && n_real >= (size_t)V;
  int grid = red_grid(ctx, vec ? n_real / V : n_real);
  if (vec)
    reduce_kernel<T, CX, true, F><<<grid, RED_THREADS, 0, st>>>(f, (const T*)x, (const T*)y, n_real, ctx->red_partials, ctx->tickets, out);
  else
    reduce_kernel<T, CX, false, F><<<grid, RED_THREADS, 0, st>>>(f, (const T*)x, (const T*)y, n_real, ctx->red_partials, ctx->tickets, out);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

template <typename F>
int dispatch_reduce(b2_ctx* ctx, F f, const void* x, const void* y, size_t n, int dtype,
                    double* out, cudaStream_t st) {
  return b2_dispatch(dtype, [&](auto t) {
    constexpr bool CX = b2_is_cx_v<decltype(t)>;
    return launch_reduce<b2_real_t<decltype(t)>, CX, F>(ctx, f, x, y, CX ? 2 * n : n, out, st);
  });
}

__global__ void zero_out_kernel(double* out, int k, double v) {
  if ((int)threadIdx.x < k) out[threadIdx.x] = v;
}

// ---- k real/complex dots in one launch ---------------------------------------
struct MultiPtrs {
  const void* x[4];
  const void* y[4];
};

template <typename T, bool CX, bool CONJ, int K>
__global__ void __launch_bounds__(RED_THREADS)
dot_multi_kernel(MultiPtrs p, size_t n_real, double* __restrict__ partials,
                 unsigned int* __restrict__ ticket, double* __restrict__ out) {
  constexpr int PER = CX ? 2 : 1;
  constexpr int NOUT = K * PER;
  double acc[NOUT];
#pragma unroll
  for (int k = 0; k < NOUT; ++k) acc[k] = 0.0;
  DotF<CONJ> f{0.0};
  const size_t stride = (size_t)gridDim.x * RED_THREADS;
  if (!CX) {
    for (size_t i = (size_t)blockIdx.x * RED_THREADS + threadIdx.x; i < n_real; i += stride) {
#pragma unroll
      for (int k = 0; k < K; ++k)
        f.real(acc + k, ((const T*)p.x[k])[i], ((const T*)p.y[k])[i]);
    }
  } else {
    const size_t nc = n_real / 2;
    for (size_t i = (size_t)blockIdx.x * RED_THREADS + threadIdx.x; i < nc; i += stride) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const T* xx = (const T*)p.x[k];
        const T* yy = (const T*)p.y[k];
        f.cx(acc + 2 * k, xx[2 * i], xx[2 * i + 1], yy[2 * i], yy[2 * i + 1]);
      }
    }
  }
  b2_grid_fold<NOUT, RED_SUM>(acc, partials, ticket, out);
}

template <typename T, bool CX, bool CONJ>
int launch_multi(b2_ctx* ctx, int k, const MultiPtrs& p, size_t n_real, double* out,
                 cudaStream_t st) {
  int grid = red_grid(ctx, n_real);
  switch (k) {
    case 1: dot_multi_kernel<T, CX, CONJ, 1><<<grid, RED_THREADS, 0, st>>>(p, n_real, ctx->red_partials, ctx->tickets, out); break;
    case 2: dot_multi_kernel<T, CX, CONJ, 2><<<grid, RED_THREADS, 0, st>>>(p, n_real, ctx->red_partials, ctx->tickets, out); break;
    case 3: dot_multi_kernel<T, CX, CONJ, 3><<<grid, RED_THREADS, 0, st>>>(p, n_real, ctx->red_partials, ctx->tickets, out); break;
    case 4: dot_multi_kernel<T, CX, CONJ, 4><<<grid, RED_THREADS, 0, st>>>(p, n_real, ctx->red_partials, ctx->tickets, out); break;
    default: return B2_ERR_ARG;
  }
  B2_LAUNCH_CHECK();
  return B2_OK;
}

}  // namespace

extern "C" int b2_dot(b2_ctx* ctx, const void* x, const void* y, size_t n, int dtype, int conj_x,
                      double* out_dev, void* stream) {
  if (!ctx || !out_dev) return B2_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (n && (!x || !y)) return B2_ERR_ARG;  // n == 0 (a rank owning no elements) runs one CTA that reads nothing
  const bool cx = (dtype == B2_C64 || dtype == B2_C128);
  if (!cx) {  // imaginary part of a real dot is 0
    zero_out_kernel<<<1, 32, 0, st>>>(out_dev, 2, 0.0);
    B2_LAUNCH_CHECK();
  }
  if (conj_x) return dispatch_reduce(ctx, DotF<true>{0.0}, x, y, n, dtype, out_dev, st);
  return dispatch_reduce(ctx, DotF<false>{0.0}, x, y, n, dtype, out_dev, st);
}

extern "C" int b2_norm_partial(b2_ctx* ctx, const void* x, size_t n, int dtype, int kind,
                               double p, double* out_dev, void* stream) {
  if (!ctx || !out_dev) return B2_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (n && !x) return B2_ERR_ARG;  // n == 0 folds to the identity: 0, or +inf for the minimum
  switch (kind) {
    case B2_NRM_COUNT_NONZERO: return dispatch_reduce(ctx, CountNzF{0.0}, x, nullptr, n, dtype, out_dev, st);
    case B2_NRM_SUM_ABS: return dispatch_reduce(ctx, SumAbsF{0.0}, x, nullptr, n, dtype, out_dev, st);
    case B2_NRM_SUM_SQ: return dispatch_reduce(ctx, SumSqF{0.0}, x, nullptr, n, dtype, out_dev, st);
    case B2_NRM_MAX_ABS: return dispatch_reduce(ctx, ExtAbsF<RED_MAX>{0.0}, x, nullptr, n, dtype, out_dev, st);
    case B2_NRM_MIN_ABS: return dispatch_reduce(ctx, ExtAbsF<RED_MIN>{0.0}, x, nullptr, n, dtype, out_dev, st);
    case B2_NRM_SUM_POW: return dispatch_reduce(ctx, SumPowF{p}, x, nullptr, n, dtype, out_dev, st);
    default: return B2_ERR_ARG;
  }
}

extern "C" int b2_dot_multi(b2_ctx* ctx, int k, const void* const* xs, const void* const* ys,
                            size_t n, int dtype, int conj_x, double* out_dev, void* stream) {
  if (!ctx || !out_dev || !xs || !ys || k < 1 || k > 4) return B2_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  // the kernel writes exactly the slots this dtype's layout uses (k doubles for real dtypes, k (re, im) pairs for
  // complex) -- the caller packs other scalars right behind them; n == 0 (a rank owning no elements) writes zeros
  MultiPtrs p;
  for (int i = 0; i < k; ++i) {
    p.x[i] = xs[i];
    p.y[i] = ys[i];
  }
  return b2_dispatch(dtype, [&](auto t) {
    using R = b2_real_t<decltype(t)>;
    constexpr bool CX = b2_is_cx_v<decltype(t)>;
    if constexpr (CX) {
      if (conj_x) return launch_multi<R, true, true>(ctx, k, p, 2 * n, out_dev, st);
    }
    return launch_multi<R, CX, false>(ctx, k, p, CX ? 2 * n : n, out_dev, st);
  });
}

// ---- device-resident scalar arithmetic for solver recurrences ------------------------
// out = num / (den1 + alpha * den2)   (den2 may be NULL): CGLS step length
// a = kold / (q.q + damp * c.c) and ratio b = k / kold (cls_basic.py:389, 395) without a host round trip
namespace {
__global__ void scalar_div_kernel(double* out, const double* num, const double* den1, const double* den2,
                                  double alpha) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    double d = *den1;
    if (den2) d += alpha * (*den2);
    *out = fabs(*num / d);
  }
}
}  // namespace

extern "C" int b2_scalar_div(double* out_dev, const double* num_dev, const double* den1_dev,
                             const double* den2_dev, double alpha, void* stream) {
  if (!out_dev || !num_dev || !den1_dev) return B2_ERR_ARG;
  scalar_div_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(out_dev, num_dev, den1_dev, den2_dev, alpha);
  B2_LAUNCH_CHECK();
  return B2_OK;
}


// history of solver scalars kept ON THE DEVICE: hist[it * nvals + j] = |src[j * stride]|, then an optional scalar copy
// (*copy_dst = *copy_src: kold <- k of the CGLS recurrence, cls_basic.py:397) and ++(*it).  Lets a whole block of CGLS
// iterations run (or replay as a CUDA graph) with no host round trip; the host reads the history once per block
// (the reference synchronises five times per iteration, cls_basic.py:389-401).
namespace {
__global__ void history_push_kernel(const double* src, int nvals, int stride, double* hist, unsigned long long* it,
                                    unsigned long long cap, double* copy_dst, const double* copy_src) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const unsigned long long i = *it;
    if (i < cap)
      for (int j = 0; j < nvals; ++j) hist[i * (unsigned long long)nvals + j] = fabs(src[j * stride]);
    if (copy_dst) *copy_dst = *copy_src;
    *it = i + 1ull;
  }
}
}  // namespace

extern "C" int b2_history_push(const double* src_dev, int nvals, int stride, double* hist_dev, void* it_dev,
                               size_t cap, double* copy_dst_dev, const double* copy_src_dev, void* stream) {
  if (!src_dev || !hist_dev || !it_dev || nvals < 1 || nvals > 16 || stride < 1) return B2_ERR_ARG;
  if ((copy_dst_dev == nullptr) != (copy_src_dev == nullptr)) return B2_ERR_ARG;
  history_push_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(src_dev, nvals, stride, hist_dev, (unsigned long long*)it_dev,
                                                          (unsigned long long)cap, copy_dst_dev, copy_src_dev);
  B2_LAUNCH_CHECK();
  return B2_OK;
}


// ---- axis-wise norm partials (DistributedArray.norm(ord, axis), DistributedArray.py:688-758, 796-807) ---------------
// x viewed as [n_outer][n_axis][n_inner] (C order); out[o * n_inner + i] = reduction over the middle axis in float64
// (the reference's float_power promotion, :755): count_nonzero / sum|x| / sum|x|^2 / max|x| / min|x| / sum|x|^p.
// One thread per output element marching down the axis (coalesced along n_inner); rows with n_inner == 1 use one
// warp per output so that the contiguous axis is read with coalesced loads.
namespace {
template <typename T> __device__ __forceinline__ double abs_of(const T* p, size_t idx, bool cx) {
  if (cx) return hypot((double)p[2 * idx], (double)p[2 * idx + 1]);
  return fabs((double)p[idx]);
}
__device__ __forceinline__ double axis_init(int kind) { return kind == B2_NRM_MIN_ABS ? INFINITY : 0.0; }
__device__ __forceinline__ double axis_fold(double acc, double a, int kind, double p) {
  switch (kind) {
    case B2_NRM_COUNT_NONZERO: return acc + (a != 0.0 ? 1.0 : 0.0);
    case B2_NRM_SUM_ABS: return acc + a;
    case B2_NRM_SUM_SQ: return acc + a * a;
    case B2_NRM_MAX_ABS: return nan_max(acc, a);
    case B2_NRM_MIN_ABS: return nan_min(acc, a);
    default: return acc + pow(a, p);
  }
}
__device__ __forceinline__ double axis_merge(double a, double b, int kind) {
  return kind == B2_NRM_MAX_ABS ? nan_max(a, b) : (kind == B2_NRM_MIN_ABS ? nan_min(a, b) : a + b);
}
template <typename T>
__global__ void __launch_bounds__(256)
norm_axis_kernel(const T* __restrict__ x, size_t n_outer, size_t n_axis, size_t n_inner, bool cx, int kind, double p,
                 double* __restrict__ out) {
  const size_t total = n_outer * n_inner;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t o = e / n_inner, i = e % n_inner;
    double acc = axis_init(kind);
    for (size_t a = 0; a < n_axis; ++a) acc = axis_fold(acc, abs_of(x, (o * n_axis + a) * n_inner + i, cx), kind, p);
    out[e] = acc;
  }
}
template <typename T>
__global__ void __launch_bounds__(256)
norm_lastaxis_kernel(const T* __restrict__ x, size_t n_outer, size_t n_axis, bool cx, int kind, double p,
                     double* __restrict__ out) {
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const int lane = threadIdx.x & 31;
  for (size_t o = warp; o < n_outer; o += nwarps) {
    double acc = axis_init(kind);
    for (size_t a = lane; a < n_axis; a += 32) acc = axis_fold(acc, abs_of(x, o * n_axis + a, cx), kind, p);
    for (int s = 16; s > 0; s >>= 1) acc = axis_merge(acc, __shfl_xor_sync(0xffffffffu, acc, s), kind);
    if (lane == 0) out[o] = acc;
  }
}
}  // namespace

extern "C" int b2_norm_axis(b2_ctx* ctx, const void* x, size_t n_outer, size_t n_axis, size_t n_inner, int dtype, int kind,
                            double p, double* out_dev, void* stream) {
  if (!ctx || !out_dev) return B2_ERR_ARG;
  if (kind < B2_NRM_COUNT_NONZERO || kind > B2_NRM_SUM_POW) return B2_ERR_ARG;
  const size_t total = n_outer * n_inner;
  if (total == 0) return B2_OK;
  if (!x && n_axis) return B2_ERR_ARG;
  const bool cx = (dtype == B2_C64 || dtype == B2_C128);
  const bool dbl = (dtype == B2_F64 || dtype == B2_C128);
  if (!cx && dtype != B2_F32 && dtype != B2_F64) return B2_ERR_DTYPE;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t cap = (size_t)ctx->sm_count * 16;
  if (n_inner == 1 && n_axis >= 64) {
    size_t blocks = (n_outer * 32 + 255) / 256;
    if (blocks > cap) blocks = cap;
    if (dbl) norm_lastaxis_kernel<double><<<(unsigned)blocks, 256, 0, st>>>((const double*)x, n_outer, n_axis, cx, kind, p, out_dev);
    else norm_lastaxis_kernel<float><<<(unsigned)blocks, 256, 0, st>>>((const float*)x, n_outer, n_axis, cx, kind, p, out_dev);
  } else {
    size_t blocks = (total + 255) / 256;
    if (blocks > cap) blocks = cap;
    if (dbl) norm_axis_kernel<double><<<(unsigned)blocks, 256, 0, st>>>((const double*)x, n_outer, n_axis, n_inner, cx, kind, p, out_dev);
    else norm_axis_kernel<float><<<(unsigned)blocks, 256, 0, st>>>((const float*)x, n_outer, n_axis, n_inner, cx, kind, p, out_dev);
  }
  B2_LAUNCH_CHECK();
  return B2_OK;
}


// ---- fused solver update + norm: out = (a_scale * *a_dev) x + (b_scale * *b_dev) y  and  norm2 = sum |out|^2 ---------
// The three vector updates of a CGLS iteration (cls_basic.py:390-391, 396) each feed a reduction the recurrence needs
// right after (x.x, s.s, c.c): one pass instead of an update pass plus a reduction pass, and three launches fewer
// per iteration.  Real coefficients (device scalars), so complex arrays are processed as arrays of 2n reals; the
// squared values are accumulated in float64 from the ROUNDED stored result, i.e. the same number a separate
// b2_dot_multi pass over `out` would produce.  Deterministic fold (b2_grid_fold) like reduce_kernel.
namespace {
template <typename T>
__global__ void __launch_bounds__(RED_THREADS)
axpby_norm2_kernel(T* out, const double* a_dev, double a_scale, const T* x, const double* b_dev, double b_scale,
                   const T* y, size_t n_real, int vec, double* __restrict__ partials, unsigned int* __restrict__ ticket,
                   double* __restrict__ res, int zero_second) {
  constexpr int V = Vec16<T>::N;
  const T a = (T)(a_scale * (a_dev ? *a_dev : 1.0)), b = (T)(b_scale * (b_dev ? *b_dev : 1.0));
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * RED_THREADS;
  size_t i = (size_t)blockIdx.x * RED_THREADS + threadIdx.x;
  if (vec) {
    const size_t nvec = n_real / V;
    for (; i < nvec; i += stride) {
      const Vec16<T> vx = load_vec_coherent(x + i * V), vy = load_vec_coherent(y + i * V);
      Vec16<T> o;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        o.v[k] = a * vx.v[k] + b * vy.v[k];
        acc = fma((double)o.v[k], (double)o.v[k], acc);
      }
      store_vec(out + i * V, o);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0)
      for (size_t t = nvec * V; t < n_real; ++t) {
        const T o = a * x[t] + b * y[t];
        out[t] = o;
        acc = fma((double)o, (double)o, acc);
      }
  } else {
    for (; i < n_real; i += stride) {
      const T o = a * x[i] + b * y[i];
      out[i] = o;
      acc = fma((double)o, (double)o, acc);
    }
  }
  // the imaginary slot of complex data is zeroed by the thread that writes res[0], after every CTA has read *a_dev
  // and *b_dev
  b2_grid_fold<1, RED_SUM>(&acc, partials, ticket, res, [&] {
    if (zero_second) res[1] = 0.0;
  });
}
}  // namespace

extern "C" int b2_lincomb_dev_norm2(b2_ctx* ctx, void* out, const double* a_dev, double a_scale, const void* x,
                                    const double* b_dev, double b_scale, const void* y, size_t n, int dtype,
                                    double* norm2_dev, void* stream) {
  if (!ctx || !norm2_dev) return B2_ERR_ARG;
  const bool cx = (dtype == B2_C64 || dtype == B2_C128);
  const bool dbl = (dtype == B2_F64 || dtype == B2_C128);
  if (!cx && dtype != B2_F32 && dtype != B2_F64) return B2_ERR_DTYPE;
  cudaStream_t st = (cudaStream_t)stream;
  if (n && (!out || !x || !y)) return B2_ERR_ARG;  // n == 0 runs one CTA that reads no array and writes norm2 = 0
  const size_t n_real = cx ? 2 * n : n;
  const int V = dbl ? 2 : 4;
  const int vec = (b2_aligned16(out) && b2_aligned16(x) && b2_aligned16(y) && n_real >= (size_t)V) ? 1 : 0;
  const int grid = red_grid(ctx, vec ? n_real / V : n_real);
  if (dbl)
    axpby_norm2_kernel<double><<<grid, RED_THREADS, 0, st>>>((double*)out, a_dev, a_scale, (const double*)x, b_dev, b_scale,
                                                            (const double*)y, n_real, vec, ctx->red_partials, ctx->tickets,
                                                            norm2_dev, cx ? 1 : 0);
  else
    axpby_norm2_kernel<float><<<grid, RED_THREADS, 0, st>>>((float*)out, a_dev, a_scale, (const float*)x, b_dev, b_scale,
                                                           (const float*)y, n_real, vec, ctx->red_partials, ctx->tickets,
                                                           norm2_dev, cx ? 1 : 0);
  B2_LAUNCH_CHECK();
  return B2_OK;
}
