// The stationary 2-D correlation core shared by nsconvolve2d.cu and nsfilters.cu: the CTA shape, the shared window
// layout, pylops' bilinear supports and weights per axis, and the register sliding window along z.  A CTA of
// N2_THREADS owns N2_TX x N2_TZ outputs; lane l of warp g owns outputs (l, 8 g .. 8 g + 7).
#pragma once
#include "common.cuh"

namespace {

constexpr int N2_LANES = 32, N2_GROUPS = 8, N2_THREADS = N2_LANES * N2_GROUPS;
constexpr int N2_RT = 8;                                   // consecutive z outputs per thread
constexpr int N2_TX = N2_LANES, N2_TZ = N2_GROUPS * N2_RT;   // outputs per CTA: 32 (x) x 64 (z)
constexpr int N2_KC = 32;                                  // taps per chunk along each axis (a multiple of N2_RT)
constexpr int N2_WR = N2_TX + N2_KC - 1;                   // window rows (x)
constexpr int N2_WC = N2_TZ + N2_KC;                       // window columns (z): the register window reads one past
constexpr int N2_WS = N2_WC + 1;                           // odd row stride: the lanes' rows fall in different banks
constexpr int N2_WELEMS = (N2_WR * N2_WS + 15) / 16 * 16;  // window elements, padded so the taps stay vector-aligned

struct Axis {
  long long n, oh, dh;
  int nf, nh, hc;
};

__device__ __forceinline__ long long floor_div(long long a, long long b) {   // b > 0
  const long long q = a / b;
  return (a % b != 0 && a < 0) ? q - 1 : q;
}

// [lo, hi): the samples of [0, n) with a non-zero weight on filter a
__host__ __device__ __forceinline__ void support(const Axis& A, int a, long long& lo, long long& hi) {
  lo = a == 0 ? 0 : A.oh + (long long)(a - 1) * A.dh + 1;
  hi = a == A.nf - 1 ? A.n : A.oh + (long long)(a + 1) * A.dh;
  lo = max(lo, 0LL);
  hi = min(hi, A.n);
}

// the float64 weight of filter a at sample j
__device__ __forceinline__ double axis_weight(const Axis& A, int a, long long j) {
  const double v = (double)(j - A.oh) / (double)A.dh;
  const double fl = floor(v);
  if (fl < 0.0) return a == 0 ? 1.0 : 0.0;
  if (fl >= (double)(A.nf - 1)) return a == A.nf - 1 ? 1.0 : 0.0;
  const int l = (int)fl;
  if (a == l) return 1.0 - (v - fl);
  return a == l + 1 ? v - fl : 0.0;
}

// out[r] += sum_(qx < nqx, qz < nqz8) hk[qx][qz] w[lane + qx][t0 + r + qz]
template <typename T>
__device__ __forceinline__ void correlate(T (&out)[N2_RT], const T* __restrict__ w, const T* __restrict__ hk, int nqx,
                                          int nqz8, int lane, int t0) {
  using VA = VecN<T, N2_RT>;
  for (int qx = 0; qx < nqx; ++qx) {
    const T* wr = w + (lane + qx) * N2_WS + t0;
    const T* hr = hk + qx * N2_KC;
    T lo[N2_RT];
#pragma unroll
    for (int r = 0; r < N2_RT; ++r) lo[r] = wr[r];
    for (int q0 = 0; q0 < nqz8; q0 += N2_RT) {
      T hi[N2_RT];
#pragma unroll
      for (int r = 0; r < N2_RT; ++r) hi[r] = wr[q0 + N2_RT + r];
      const VA hv = *reinterpret_cast<const VA*>(hr + q0);
#pragma unroll
      for (int qq = 0; qq < N2_RT; ++qq) {
#pragma unroll
        for (int r = 0; r < N2_RT; ++r) out[r] = fma(hv.v[qq], r + qq < N2_RT ? lo[r + qq] : hi[r + qq - N2_RT], out[r]);
      }
#pragma unroll
      for (int r = 0; r < N2_RT; ++r) lo[r] = hi[r];
    }
  }
}

}  // namespace
