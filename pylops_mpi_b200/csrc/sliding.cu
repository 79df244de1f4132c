// Tapered overlap-add of windows: the combining stage of pylops.signalprocessing.Sliding2D / Sliding3D (pylops 2.x,
// HStack of Restriction.H over BlockDiag of Diagonal(taper) * Op), on the window geometry of sliding.cuh.
//
// Windows [nw0][nw1][len0][len1][inner], data [n0][n1][inner] (inner = nt * n_inner values per trace, n_inner 2 for
// the (re, im) pairs of complex data), taper table [nw0 * nw1][len0][len1] of the data's type (NULL: no taper).
//   forward (fold):    d[a][b][k] = sum over i0 of (sum over i1 of tap[w][a - i0 step0][b - i1 step1] * win[w][..][k])
//                      over the windows that hold trace (a, b), both sums ascending; 0 where no window holds it
//   adjoint (unfold):  win[w][j0][j1][k] = tap[w][j0][j1] * d[i0 step0 + j0][i1 step1 + j1][k]
// One thread per output value, so no atomics and no workspace: one launch per call, the same bits on every run.
#include "sliding.cuh"

namespace {

constexpr int SL_THREADS = 256;
constexpr unsigned SL_MAX_BLOCKS = 1u << 16;

template <typename T>
__global__ void __launch_bounds__(SL_THREADS)
fold_kernel(const T* __restrict__ win, T* __restrict__ d, long long total, long long inner, Windows g,
            const T* __restrict__ tap) {
  for (long long i = (long long)blockIdx.x * SL_THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * SL_THREADS) {
    const long long tr = i / inner, k = i - tr * inner;
    const long long a = tr / g.n1, b = tr - a * g.n1;
    long long f0, l0, f1, l1;
    covering(a, g.nw0, g.len0, g.step0, f0, l0);
    covering(b, g.nw1, g.len1, g.step1, f1, l1);
    T out = T(0);
    for (long long i0 = f0; i0 <= l0; ++i0) {
      T part = T(0);
      for (long long i1 = f1; i1 <= l1; ++i1) {
        const long long w = i0 * g.nw1 + i1;
        const long long t = (w * g.len0 + a - i0 * g.step0) * g.len1 + b - i1 * g.step1;
        const T v = __ldg(win + t * inner + k);
        part = add_rn(part, tap ? mul_rn(__ldg(tap + t), v) : v);
      }
      out = add_rn(out, part);
    }
    d[i] = out;
  }
}

template <typename T>
__global__ void __launch_bounds__(SL_THREADS)
unfold_kernel(const T* __restrict__ d, T* __restrict__ win, long long total, long long inner, Windows g,
              const T* __restrict__ tap) {
  for (long long i = (long long)blockIdx.x * SL_THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * SL_THREADS) {
    const long long t = i / inner, k = i - t * inner;        // t = (w * len0 + j0) * len1 + j1
    const long long r = t / g.len1, j1 = t - r * g.len1;
    const long long w = r / g.len0, j0 = r - w * g.len0;
    const long long i0 = w / g.nw1, i1 = w - i0 * g.nw1;
    const T v = __ldg(d + ((i0 * g.step0 + j0) * g.n1 + i1 * g.step1 + j1) * inner + k);
    win[i] = tap ? mul_rn(__ldg(tap + t), v) : v;
  }
}

}  // namespace

extern "C" int b2_sliding(b2_ctx* ctx, const void* x, void* y, size_t n0, size_t n1, size_t nt, size_t n_inner,
                          size_t nwins0, size_t nwins1, size_t nwin0, size_t nwin1, size_t step0, size_t step1,
                          const void* tap, int adjoint, int dtype, void* stream) {
  if (!ctx || !x || !y || x == y) return B2_ERR_ARG;
  Windows g;
  if (!make_windows(n0, n1, nwins0, nwins1, nwin0, nwin1, step0, step1, g)) return B2_ERR_ARG;
  const size_t axis_max = (size_t)1 << 31;
  if (nt == 0 || nt >= axis_max || n_inner == 0 || n_inner >= axis_max) return B2_ERR_ARG;
  const long long inner = (long long)(nt * n_inner);
  using u128 = unsigned __int128;
  const u128 nwv = (u128)(nwins0 * nwin0) * (u128)(nwins1 * nwin1), ndv = (u128)n0 * n1;   // window, data traces
  if ((nwv > ndv ? nwv : ndv) * inner >= ((u128)1 << 62)) return B2_ERR_ARG;
  const long long total = adjoint ? g.nw0 * g.nw1 * g.len0 * g.len1 * inner : g.n0 * g.n1 * inner;
  const long long want = (total + SL_THREADS - 1) / SL_THREADS;
  const unsigned blocks = (unsigned)(want < (long long)SL_MAX_BLOCKS ? want : SL_MAX_BLOCKS);
  return b2_dispatch_real(dtype, [&](auto t) -> int {
    using T = decltype(t);
    const T* xs = static_cast<const T*>(x);
    T* ys = static_cast<T*>(y);
    const T* tp = static_cast<const T*>(tap);
    if (adjoint)
      unfold_kernel<T><<<blocks, SL_THREADS, 0, (cudaStream_t)stream>>>(xs, ys, total, inner, g, tp);
    else
      fold_kernel<T><<<blocks, SL_THREADS, 0, (cudaStream_t)stream>>>(xs, ys, total, inner, g, tp);
    B2_LAUNCH_CHECK();
    return B2_OK;
  });
}
