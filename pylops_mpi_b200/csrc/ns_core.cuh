// The core shared by the non-stationary kernels nsconvolve2d.cu, nsconvolve3d.cu and nsfilters.cu: the thread layout
// of a CTA, pylops' bilinear supports and weights per axis, the filters and taps a tile can reach, and the register
// sliding-window correlation.  A CTA of NS_THREADS threads runs lanes along its row axis (one output row each, every
// tap a broadcast); lane l of warp g owns the NS_RT consecutive z outputs 8 g .. 8 g + 7 of row l.  The axis geometry
// is templated on the coordinate type I: 64-bit in 2-D, 32-bit in 3-D, whose three axes would not fit the registers
// in 64 bits.
#pragma once
#include "common.cuh"

namespace {

constexpr int NS_LANES = 32, NS_GROUPS = 8, NS_THREADS = NS_LANES * NS_GROUPS;
constexpr int NS_RT = 8;                                   // consecutive z outputs per thread
constexpr int NS_TZ = NS_GROUPS * NS_RT;                   // z outputs per CTA row: 64

// the 2-D tile of nsconvolve2d.cu and nsfilters.cu
constexpr int N2_TX = NS_LANES;                            // outputs per CTA: 32 (x) x 64 (z)
constexpr int N2_KC = 32;                                  // taps per chunk along each axis (a multiple of NS_RT)
constexpr int N2_WR = N2_TX + N2_KC - 1;                   // window rows (x)
constexpr int N2_WC = NS_TZ + N2_KC;                       // window columns (z): the register window reads one past
constexpr int N2_WS = N2_WC + 1;                           // odd row stride: the lanes' rows fall in different banks
constexpr int N2_WELEMS = (N2_WR * N2_WS + 15) / 16 * 16;  // window elements, padded so the taps stay vector-aligned

// one axis: n samples, nf filters of nh taps (centre hc) at the samples oh + a dh
template <typename I>
struct AxisT {
  I n, oh, dh;
  int nf, nh, hc;
};

// the axis of n samples with nf filters of nh taps at oh + a dh; false for one the kernels refuse.  With 32-bit
// coordinates every axis, filter size and node position stays below 2^29 samples, so that no sum of two of them
// overflows (one filter takes any step: its weight is 1 everywhere)
template <typename I>
bool make_axis(size_t n, int nf, int nh, long long oh, long long dh, AxisT<I>& A) {
  if (n == 0 || nf < 1 || nh < 1 || dh < 1) return false;
  if constexpr (sizeof(I) < sizeof(long long)) {
    constexpr long long LIM = 1LL << 29;
    if (nf == 1) dh = 1;
    if (n >= (size_t)LIM || nh >= LIM || oh <= -LIM || oh >= LIM || dh >= LIM || oh + (nf - 1) * dh >= LIM)
      return false;
  }
  A = AxisT<I>{(I)n, (I)oh, (I)dh, nf, nh, nh / 2};
  return true;
}

template <typename I>
__device__ __forceinline__ I floor_div(I a, I b) {   // b > 0
  const I q = a / b;
  return (a % b != 0 && a < 0) ? q - 1 : q;
}

// [lo, hi): the samples of [0, n) with a non-zero weight on filter a
template <typename I>
__host__ __device__ __forceinline__ void support(const AxisT<I>& A, int a, I& lo, I& hi) {
  lo = a == 0 ? 0 : A.oh + (I)(a - 1) * A.dh + 1;
  hi = a == A.nf - 1 ? A.n : A.oh + (I)(a + 1) * A.dh;
  lo = max(lo, (I)0);
  hi = min(hi, A.n);
}

// the float64 weight of filter a at sample j
template <typename I>
__device__ __forceinline__ double axis_weight(const AxisT<I>& A, int a, I j) {
  const double v = (double)(j - A.oh) / (double)A.dh;
  const double fl = floor(v);
  if (fl < 0.0) return a == 0 ? 1.0 : 0.0;
  if (fl >= (double)(A.nf - 1)) return a == A.nf - 1 ? 1.0 : 0.0;
  const int l = (int)fl;
  if (a == l) return 1.0 - (v - fl);
  return a == l + 1 ? v - fl : 0.0;
}

// [af, al]: the filters whose support can meet the samples [lo, hi)
template <typename I>
__device__ __forceinline__ void filter_span(const AxisT<I>& A, I lo, I hi, int& af, int& al) {
  const I l = max(lo, (I)0), h = min(hi, A.n);
  af = (int)min(max(floor_div(l - A.oh, A.dh), (I)0), (I)A.nf - 1);
  al = (int)min(max(floor_div(h - 1 - A.oh + A.dh - 1, A.dh), (I)0), (I)A.nf - 1);
}

// taps [qlo, qhi) of filter a that can meet its support from a tile of nt outputs at i0 (window index m = sample
// jb + m)
template <typename I>
__device__ __forceinline__ bool tap_span(const AxisT<I>& A, int a, I i0, I jb, int nt, bool adj, int& qlo, int& qhi) {
  I lo, hi;
  support(A, a, lo, hi);
  I q0, q1;
  if (!adj) {                     // outputs t in [0, nt) read t + q; the non-zero inputs are the support's
    q0 = lo - jb - nt + 1;
    q1 = hi - jb;
  } else {                        // the outputs in the support read t + q; the non-zero inputs are [0, n)'s
    const I tlo = max(lo - i0, (I)0), thi = min(hi - i0, (I)nt);
    if (tlo >= thi) return false;
    q0 = -jb - thi + 1;
    q1 = A.n - jb - tlo;
  }
  q0 = max(q0, (I)0);
  q1 = min(q1, (I)A.nh);
  qlo = (int)q0;
  qhi = (int)q1;
  return q0 < q1;
}

// for every output plane t whose tap plane m - t lies in [0, nqx):
//   out[t][r] += sum_(qy < nqy, qz < nqz8) hk[m - t][qy][qz] w[lane + qy][t0 + r + qz]
// with taps in chunks of KC x KC and window rows WS apart; one window row in registers serves every such t
template <typename T, int TX, int KC, int WS>
__device__ __forceinline__ void correlate_plane(T (&out)[TX][NS_RT], const T* __restrict__ w, const T* __restrict__ hk,
                                                int m, int nqx, int nqy, int nqz8, int lane, int t0) {
  using VA = VecN<T, NS_RT>;
  for (int qy = 0; qy < nqy; ++qy) {
    const T* wr = w + (lane + qy) * WS + t0;
    T lo[NS_RT];
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) lo[r] = wr[r];
    for (int q0 = 0; q0 < nqz8; q0 += NS_RT) {
      T hi[NS_RT];
#pragma unroll
      for (int r = 0; r < NS_RT; ++r) hi[r] = wr[q0 + NS_RT + r];
#pragma unroll
      for (int t = 0; t < TX; ++t) {
        const int qx = m - t;
        if (qx < 0 || qx >= nqx) continue;
        const VA hv = *reinterpret_cast<const VA*>(hk + (qx * KC + qy) * KC + q0);
#pragma unroll
        for (int qq = 0; qq < NS_RT; ++qq) {
#pragma unroll
          for (int r = 0; r < NS_RT; ++r)
            out[t][r] = fma(hv.v[qq], r + qq < NS_RT ? lo[r + qq] : hi[r + qq - NS_RT], out[t][r]);
        }
      }
#pragma unroll
      for (int r = 0; r < NS_RT; ++r) lo[r] = hi[r];
    }
  }
}

// the 2-D tile's correlation: out[r] += sum_(qx < nqx, qz < nqz8) hk[qx][qz] w[lane + qx][t0 + r + qz]
template <typename T>
__device__ __forceinline__ void correlate(T (&out)[NS_RT], const T* __restrict__ w, const T* __restrict__ hk, int nqx,
                                          int nqz8, int lane, int t0) {
  correlate_plane<T, 1, N2_KC, N2_WS>(reinterpret_cast<T(&)[1][NS_RT]>(out), w, hk, 0, 1, nqx, nqz8, lane, t0);
}

}  // namespace
