// Window geometry of pylops.signalprocessing.Sliding1D / Sliding2D / Sliding3D / Patch2D / Patch3D, shared by the
// overlap-add kernel (sliding.cu) and the windowed Radon kernels (radon.cu).
//
// A section [n0][n1][nt] (each sample n_inner values) holds nw0 x nw1 x nw2 windows of len0 x len1 traces and len2
// samples: window (i0, i1, i2), w = (i0 * nw1 + i1) * nw2 + i2, starts at (trace i0 * step0, trace i1 * step1,
// sample i2 * step2).  Sliding2D is the case n0 = nw0 = len0 = step0 = 1, and the trace-only windows of Sliding2D /
// Sliding3D are nw2 = 1, len2 = nt; Sliding1D has windows along the samples only.  A data sample sums its windows'
// tapered values as the restated chain does: over i0 ascending, of the sum over i1 ascending, of the sum over i2
// ascending (the nested HStacks, innermost last), every product and sum in the data's type, rounded to nearest
// operation by operation.
#pragma once
#include "common.cuh"

struct Windows {
  long long n0, n1, nt, nw0, nw1, nw2, len0, len1, len2, step0, step1, step2;
};

// the windows [first, last] of one axis that hold index a (first > last: none)
__device__ __forceinline__ void covering(long long a, long long nw, long long len, long long step, long long& first,
                                         long long& last) {
  const long long lo = a - len + 1;
  first = lo <= 0 ? 0 : (lo + step - 1) / step;
  last = min(a / step, nw - 1);
}

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

// A window's taper, in two steps so that kernels which walk the samples of one window trace form the per-trace part
// once: trace(g, i0, i1, j0, j1) for window trace (j0, j1) of windows (i0, i1, *), then sample(g, that, i2, j2) for
// sample j2 of window i2, in the data's type T.
//
// TableTaper: b2_sliding's table [nw0 * nw1][len0][len1] of T, constant along the samples (windows along the traces
// only: nw2 = 1).  NULL: no taper.
template <typename T>
struct TableTaper {
  static constexpr bool time_windows = false;
  const T* tab;
  __device__ __forceinline__ bool on() const { return tab != nullptr; }
  __device__ __forceinline__ T trace(const Windows& g, long long i0, long long i1, long long j0, long long j1) const {
    return __ldg(tab + ((i0 * g.nw1 + i1) * g.len0 + j0) * g.len1 + j1);
  }
  __device__ __forceinline__ T sample(const Windows&, T tr, long long, long long) const { return tr; }
};

// AxisTaper: one float64 table [nw_a][len_a] per window axis (NULL: that axis is not tapered; all three NULL: no
// taper), formed (T)((t0 * t1) * t2) in float64 and rounded once -- the bits of pylops' float64 outer product of the
// axis tapers cast to the operator's dtype.
template <typename T>
struct AxisTaper {
  static constexpr bool time_windows = true;
  const double *t0, *t1, *t2;
  __device__ __forceinline__ bool on() const { return t0 || t1 || t2; }
  __device__ __forceinline__ double trace(const Windows& g, long long i0, long long i1, long long j0,
                                          long long j1) const {
    const double a = t0 ? __ldg(t0 + i0 * g.len0 + j0) : 1.0;
    return __dmul_rn(a, t1 ? __ldg(t1 + i1 * g.len1 + j1) : 1.0);
  }
  __device__ __forceinline__ T sample(const Windows& g, double tr, long long i2, long long j2) const {
    return (T)__dmul_rn(tr, t2 ? __ldg(t2 + i2 * g.len2 + j2) : 1.0);
  }
};

// the window geometry of an entry point's arguments, or false for a zero size, an axis of 2^31 or more, windows
// that leave the section, or 2^62 or more window or section values
static inline bool make_windows(size_t n0, size_t n1, size_t nt, size_t n_inner, size_t nw0, size_t nw1, size_t nw2,
                                size_t len0, size_t len1, size_t len2, size_t step0, size_t step1, size_t step2,
                                Windows& w) {
  const size_t axis_max = (size_t)1 << 31;
  for (size_t n : {n0, n1, nt, n_inner, nw0, nw1, nw2, len0, len1, len2, step0, step1, step2})
    if (n == 0 || n >= axis_max) return false;
  if ((nw0 - 1) * step0 + len0 > n0 || (nw1 - 1) * step1 + len1 > n1 || (nw2 - 1) * step2 + len2 > nt) return false;
  using u128 = unsigned __int128;
  const u128 lim = (u128)1 << 62;
  u128 nwv = (u128)(nw0 * len0) * (nw1 * len1), ndv = (u128)n0 * n1 * nt;   // each factor below 2^62
  if (nwv >= lim || (nwv *= nw2 * len2) >= lim || ndv >= lim || nwv * n_inner >= lim || ndv * n_inner >= lim)
    return false;
  w = {(long long)n0,  (long long)n1,   (long long)nt,    (long long)nw0,   (long long)nw1,   (long long)nw2,
       (long long)len0, (long long)len1, (long long)len2, (long long)step0, (long long)step1, (long long)step2};
  return true;
}
