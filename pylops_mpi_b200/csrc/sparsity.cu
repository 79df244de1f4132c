// Fused proximal-gradient update behind ISTA / FISTA ("next" row: pylops_mpi/optimization/cls_sparsity.py:270-343,
// 578-662).  The reference makes 8+ passes over the model per iteration (x.copy, x + grad, threshold, x - xold, two
// norms, FISTA's z update); this is ONE pass:
//     u = base + alpha * g ;  v = thresh(u) ;  xnew = v ;  znew = v + c (v - xold)
//     sums[0] = sum |v - xold|^2 ,  sums[1] = sum |v|        (local partials; the caller all-reduces them)
// HBM-bound: algorithmic bytes per element = (2..3 reads + 1..2 writes) * sizeof(T).
// Thresholds restate third-party pylops.optimization.cls_sparsity._soft/_hard/_halfthreshold (pylops 2.x).
#include <math.h>
#include "common.cuh"

namespace {

constexpr int SP_THREADS = B2_RED_THREADS;

struct SpParams {
  const void* base;
  const void* g;
  const void* xold;
  void* xnew;
  void* znew;
  double alpha, thresh, c;
  double hard_cut, half_cut;
  size_t n_real;
  int kind;
};

// element arithmetic runs in the array's own precision C (float for f32/c64 -- as the reference's NumPy does --
// double for f64/c128); only the two running sums are float64.  (A first version computed everything in
// double: the f32<->f64 conversions, not HBM, bounded it at 0.64 of the copy peak.)
template <typename C> struct M;
template <> struct M<float> {
  static __device__ __forceinline__ float abs(float x) { return fabsf(x); }
  static __device__ __forceinline__ float max(float a, float b) { return fmaxf(a, b); }
  static __device__ __forceinline__ float min(float a, float b) { return fminf(a, b); }
  static __device__ __forceinline__ float cps(float a, float b) { return copysignf(a, b); }
  static __device__ __forceinline__ float hyp(float a, float b) { return hypotf(a, b); }
  static __device__ __forceinline__ float rsq(float a) { return rsqrtf(a); }
  static __device__ __forceinline__ float acs(float a) { return acosf(a); }
  static __device__ __forceinline__ float cs(float a) { return cosf(a); }
  static __device__ __forceinline__ float fm(float a, float b, float c) { return fmaf(a, b, c); }
  // the hard cut rounded DOWN: a <= cut holds for a float a exactly when it holds in float64, as in pylops, which
  // compares |x| with np.sqrt(2 * thresh), a float64 scalar
  static __device__ __forceinline__ float cut(double c) { return __double2float_rd(c); }
};
template <> struct M<double> {
  static __device__ __forceinline__ double abs(double x) { return fabs(x); }
  static __device__ __forceinline__ double max(double a, double b) { return fmax(a, b); }
  static __device__ __forceinline__ double min(double a, double b) { return fmin(a, b); }
  static __device__ __forceinline__ double cps(double a, double b) { return copysign(a, b); }
  static __device__ __forceinline__ double hyp(double a, double b) { return hypot(a, b); }
  static __device__ __forceinline__ double rsq(double a) { return rsqrt(a); }
  static __device__ __forceinline__ double acs(double a) { return acos(a); }
  static __device__ __forceinline__ double cs(double a) { return cos(a); }
  static __device__ __forceinline__ double fm(double a, double b, double c) { return fma(a, b, c); }
  static __device__ __forceinline__ double cut(double c) { return c; }
};

template <typename C>
struct SpConst {  // per-thread copies of the scalars in precision C
  C alpha, thresh, c, hard_cut, half_cut;
  int kind;
};

template <typename C>
__device__ __forceinline__ C thr_real(C u, const SpConst<C>& k) {
  const C a = M<C>::abs(u);
  switch (k.kind) {
    case B2_THRESH_SOFT: {  // max(a - t, 0) that keeps a NaN, as np.maximum does (fmax would return 0)
      const C d = a - k.thresh;
      return M<C>::cps(d <= (C)0 ? (C)0 : d, u);
    }
    case B2_THRESH_HARD: return a <= k.hard_cut ? (C)0 : u;
    case B2_THRESH_HALF: {
      if (a <= k.half_cut) return (C)0;
      const C r = M<C>::rsq(a * (C)(1.0 / 3.0));  // (a/3)^-1.5 = rsqrt(a/3)^3
      C arg = (k.thresh * (C)0.125) * (r * r * r);
      arg = M<C>::min(M<C>::max(arg, (C)-1), (C)1);
      const C phi = (C)(2.0 / 3.0) * M<C>::acs(arg);
      return (C)(2.0 / 3.0) * u * ((C)1 + M<C>::cs((C)(2.0 * 3.14159265358979323846 / 3.0) - phi));
    }
    default: return u;
  }
}
// returns |v| of the thresholded value (one hypot per element serves the threshold and the l1 sum)
template <typename C>
__device__ __forceinline__ C thr_cx(C& ur, C& ui, const SpConst<C>& k) {
  const C a = M<C>::hyp(ur, ui);
  C s = (C)1;
  if (k.kind == B2_THRESH_SOFT) {  // a NaN |u| gives s = NaN, so both components come out NaN, as in pylops
    const C d = a - k.thresh;
    s = d <= (C)0 ? (C)0 : d / a;
  }
  else if (k.kind == B2_THRESH_HARD) s = a <= k.hard_cut ? (C)0 : (C)1;
  ur *= s;
  ui *= s;
  return a * s;
}

// one "item" = 1 real scalar or 1 complex pair; acc[0] += |v - xold|^2, acc[1] += |v| (precision T, folded into
// float64 once per 16-byte vector by the caller)
template <typename T, bool CX>
__device__ __forceinline__ void item(const SpConst<T>& k, const T* b, const T* g, const T* xo, T* xn, T* zn,
                                     bool has_g, bool has_xo, bool has_zn, T* acc) {
  if (!CX) {
    T u = b[0];
    if (has_g) u = M<T>::fm(k.alpha, g[0], u);
    const T v = thr_real<T>(u, k);
    const T d = has_xo ? v - xo[0] : (T)0;
    xn[0] = v;
    if (has_zn) zn[0] = M<T>::fm(k.c, d, v);
    acc[0] = M<T>::fm(d, d, acc[0]);
    acc[1] += M<T>::abs(v);
  } else {
    T ur = b[0], ui = b[1];
    if (has_g) { ur = M<T>::fm(k.alpha, g[0], ur); ui = M<T>::fm(k.alpha, g[1], ui); }
    const T av = thr_cx<T>(ur, ui, k);
    const T dr = has_xo ? ur - xo[0] : (T)0, di = has_xo ? ui - xo[1] : (T)0;
    xn[0] = ur; xn[1] = ui;
    if (has_zn) { zn[0] = M<T>::fm(k.c, dr, ur); zn[1] = M<T>::fm(k.c, di, ui); }
    acc[0] += dr * dr + di * di;
    acc[1] += av;
  }
}

constexpr int SP_UNROLL = 4;

template <typename T, bool CX, bool VEC>
__global__ void __launch_bounds__(SP_THREADS)
sparse_update_kernel(const __grid_constant__ SpParams p, double* __restrict__ partials,
                     unsigned int* __restrict__ ticket, double* __restrict__ out) {
  constexpr int V = Vec16<T>::N;
  constexpr int STEP = CX ? 2 : 1;
  const T* base = (const T*)p.base;
  const T* g = (const T*)p.g;
  const T* xo = (const T*)p.xold;
  T* xn = (T*)p.xnew;
  T* zn = (T*)p.znew;
  const bool has_g = g != nullptr, has_xo = xo != nullptr, has_zn = zn != nullptr;
  const bool xo_is_base = xo == base;
  SpConst<T> k;
  k.alpha = (T)p.alpha; k.thresh = (T)p.thresh; k.c = (T)p.c; k.hard_cut = M<T>::cut(p.hard_cut); k.half_cut = (T)p.half_cut;
  k.kind = p.kind;
  double acc[2] = {0.0, 0.0};
  const size_t stride = (size_t)gridDim.x * SP_THREADS;
  size_t i = (size_t)blockIdx.x * SP_THREADS + threadIdx.x;
  if (VEC) {
    const size_t nvec = p.n_real / V;
    // coherent loads throughout: xnew / znew may alias base / xold (in-place update); every element is read
    // and written by the same thread, loads of an unrolled group all precede its stores
    for (; i + (SP_UNROLL - 1) * stride < nvec; i += SP_UNROLL * stride) {
      Vec16<T> vb[SP_UNROLL], vg[SP_UNROLL], vo[SP_UNROLL];
#pragma unroll
      for (int u = 0; u < SP_UNROLL; ++u) vb[u] = load_vec_coherent(base + (i + u * stride) * V);
      if (has_g) {
#pragma unroll
        for (int u = 0; u < SP_UNROLL; ++u) vg[u] = load_vec_coherent(g + (i + u * stride) * V);
      }
      if (has_xo && !xo_is_base) {
#pragma unroll
        for (int u = 0; u < SP_UNROLL; ++u) vo[u] = load_vec_coherent(xo + (i + u * stride) * V);
      }
#pragma unroll
      for (int u = 0; u < SP_UNROLL; ++u) {
        Vec16<T> vx, vz;
        T a2[2] = {(T)0, (T)0};
        const Vec16<T>& vold = xo_is_base ? vb[u] : vo[u];
#pragma unroll
        for (int e = 0; e < V; e += STEP)
          item<T, CX>(k, vb[u].v + e, vg[u].v + e, vold.v + e, vx.v + e, vz.v + e, has_g, has_xo, has_zn, a2);
        acc[0] += (double)a2[0];
        acc[1] += (double)a2[1];
        store_vec(xn + (i + u * stride) * V, vx);
        if (has_zn) store_vec(zn + (i + u * stride) * V, vz);
      }
    }
    for (; i < nvec; i += stride) {
      Vec16<T> vb = load_vec_coherent(base + i * V), vg = vb, vo = vb, vx, vz;
      if (has_g) vg = load_vec_coherent(g + i * V);
      if (has_xo && !xo_is_base) vo = load_vec_coherent(xo + i * V);
      T a2[2] = {(T)0, (T)0};
#pragma unroll
      for (int e = 0; e < V; e += STEP)
        item<T, CX>(k, vb.v + e, vg.v + e, vo.v + e, vx.v + e, vz.v + e, has_g, has_xo, has_zn, a2);
      acc[0] += (double)a2[0];
      acc[1] += (double)a2[1];
      store_vec(xn + i * V, vx);
      if (has_zn) store_vec(zn + i * V, vz);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      for (size_t t = nvec * V; t + STEP - 1 < p.n_real; t += STEP) {
        T a2[2] = {(T)0, (T)0};
        item<T, CX>(k, base + t, g + t, xo + t, xn + t, zn + t, has_g, has_xo, has_zn, a2);
        acc[0] += (double)a2[0];
        acc[1] += (double)a2[1];
      }
    }
  } else {
    const size_t nit = p.n_real / STEP;
    for (; i < nit; i += stride) {
      const size_t t = i * STEP;
      T a2[2] = {(T)0, (T)0};
      item<T, CX>(k, base + t, g + t, xo + t, xn + t, zn + t, has_g, has_xo, has_zn, a2);
      acc[0] += (double)a2[0];
      acc[1] += (double)a2[1];
    }
  }
  b2_grid_fold<2, RED_SUM>(acc, partials, ticket, out);
}

template <typename T, bool CX>
int launch(b2_ctx* ctx, const SpParams& p, double* sums, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  const bool vec = b2_aligned16(p.base) && b2_aligned16(p.g) && b2_aligned16(p.xold) && b2_aligned16(p.xnew) &&
                   b2_aligned16(p.znew) && p.n_real >= (size_t)V;
  const int grid = b2_red_grid(ctx, vec ? p.n_real / V : p.n_real, SP_THREADS * SP_UNROLL);
  if (vec)
    sparse_update_kernel<T, CX, true><<<grid, SP_THREADS, 0, st>>>(p, ctx->red_partials, ctx->tickets, sums);
  else
    sparse_update_kernel<T, CX, false><<<grid, SP_THREADS, 0, st>>>(p, ctx->red_partials, ctx->tickets, sums);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

}  // namespace

extern "C" int b2_sparse_update(b2_ctx* ctx, const void* base, const void* g, double alpha, const void* xold,
                                double thresh, int kind, void* xnew, void* znew, double c, double* sums_dev,
                                size_t n, int dtype, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (kind < B2_THRESH_NONE || kind > B2_THRESH_HALF || thresh < 0.0) return B2_ERR_ARG;
  const bool cx = dtype == B2_C64 || dtype == B2_C128;
  if (cx && kind == B2_THRESH_HALF) return B2_ERR_UNSUPPORTED;
  if (b2_dtype_size(dtype) == 0 || dtype == B2_BF16 || dtype == B2_I64) return B2_ERR_DTYPE;
  // a rank may own no model elements (n == 0, null arrays allowed): one CTA reads nothing and writes zero sums
  // (if sums_dev is given), which are still all-reduced
  if (n && (!base || !xnew || (znew && !xold))) return B2_ERR_ARG;
  SpParams p;
  p.base = base; p.g = g; p.xold = xold; p.xnew = xnew; p.znew = znew;
  p.alpha = alpha; p.thresh = thresh; p.c = c; p.kind = kind;
  p.hard_cut = sqrt(2.0 * thresh);
  p.half_cut = (pow(54.0, 1.0 / 3.0) / 4.0) * pow(thresh, 2.0 / 3.0);  // pylops' 54 ** (1/3), not cbrt(54)
  p.n_real = cx ? 2 * n : n;
  cudaStream_t st = (cudaStream_t)stream;
  return b2_dispatch(dtype, [&](auto t) {
    return launch<b2_real_t<decltype(t)>, b2_is_cx_v<decltype(t)>>(ctx, p, sums_dev, st);
  });
}
