// The first derivative of pylops.avo.poststack.PoststackLinearModelling (FirstDerivative, edge=False, sampling=1)
// as the fused convolution kernels apply it to values already in registers or shared memory: the stencil kernel's
// arithmetic (stencil.cu: non-zero taps in ascending offset order, each an fma into an accumulator that starts at 0),
// so that a fused kernel equals b2_derivative_axis followed (or preceded) by its convolution bit for bit.
#pragma once
#include "common.cuh"

// Compile-time derivative stage of a convolution kernel: none, D before C (y = C D x), D^T after C^T (x = D^T C^T y)
constexpr int DS_NONE = 0, DS_FWD = 1, DS_ADJ = 2;
template <int DS>
struct DsTag { static constexpr int value = DS; };

// f(T(), DsTag<DS>()) for the real dtype (B2_ERR_DTYPE for any other) and the stage of a plain (fused == false) or
// derivative-fused launch
template <typename F>
int ds_dispatch(int dtype, bool fused, int adjoint, F f) {
  const auto stage = [&](auto t) {
    return !fused ? f(t, DsTag<DS_NONE>()) : adjoint ? f(t, DsTag<DS_ADJ>()) : f(t, DsTag<DS_FWD>());
  };
  return b2_dispatch_real(dtype, stage);
}

// (D x)[j] from x[j-1], x[j], x[j+1] on a line of n samples: 0.5 (x[j+1] - x[j-1]) on [1, n-2] (centered) or
// x[j+1] - x[j] on [0, n-2] (forward), zero elsewhere
template <typename T>
__device__ __forceinline__ T fd_fwd(T xm, T x0, T xp, long long j, long long n, int kind) {
  T acc = T(0);
  if (kind == B2_FD_CENTERED) {
    if (j >= 1 && j <= n - 2) { acc = fma(T(-0.5), xm, acc); acc = fma(T(0.5), xp, acc); }
  } else if (j >= 0 && j <= n - 2) {
    acc = fma(T(-1), x0, acc);
    acc = fma(T(1), xp, acc);
  }
  return acc;
}

// (D^T e)[i] from e[i-1], e[i], e[i+1]: row i of the transpose, whose taps come from the forward rows i-1, i, i+1
template <typename T>
__device__ __forceinline__ T fd_adj(T em, T e0, T ep, long long i, long long n, int kind) {
  T acc = T(0);
  if (kind == B2_FD_CENTERED) {
    if (i - 1 >= 1 && i - 1 <= n - 2) acc = fma(T(0.5), em, acc);
    if (i + 1 >= 1 && i + 1 <= n - 2) acc = fma(T(-0.5), ep, acc);
  } else {
    if (i >= 1 && i - 1 <= n - 2) acc = fma(T(1), em, acc);
    if (i <= n - 2) acc = fma(T(-1), e0, acc);
  }
  return acc;
}
