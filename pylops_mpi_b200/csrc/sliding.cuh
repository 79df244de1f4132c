// Window geometry of pylops.signalprocessing.Sliding2D / Sliding3D, shared by the overlap-add kernel (sliding.cu) and
// the windowed Radon kernels (radon.cu).
//
// A section [n0][n1][...] holds nw0 x nw1 windows of len0 x len1 traces: window (i0, i1), w = i0 * nw1 + i1, starts
// at trace (i0 * step0, i1 * step1).  Sliding2D is the case n0 = nw0 = len0 = step0 = 1.  A data sample sums its
// windows' tapered values as the restated chain does: for each i0 ascending the sum over i1 ascending (the inner
// HStack), added to the sum over i0 (the outer HStack), every product and sum in the data's type, rounded to nearest
// operation by operation.
#pragma once
#include "common.cuh"

struct Windows {
  long long n0, n1, nw0, nw1, len0, len1, step0, step1;
};

// the windows [first, last] of one axis that hold trace a (first > last: none)
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

// the window geometry of an entry point's arguments, or false for a zero size, an axis of 2^31 or more, or windows
// that leave the section
static inline bool make_windows(size_t n0, size_t n1, size_t nw0, size_t nw1, size_t len0, size_t len1, size_t step0,
                                size_t step1, Windows& w) {
  const size_t axis_max = (size_t)1 << 31;
  for (size_t n : {n0, n1, nw0, nw1, len0, len1, step0, step1})
    if (n == 0 || n >= axis_max) return false;
  if ((nw0 - 1) * step0 + len0 > n0 || (nw1 - 1) * step1 + len1 > n1) return false;
  w = {(long long)n0, (long long)n1, (long long)nw0, (long long)nw1, (long long)len0, (long long)len1,
       (long long)step0, (long long)step1};
  return true;
}
