// Tapered overlap-add of windows: the combining stage of pylops.signalprocessing.Sliding1D / Sliding2D / Sliding3D /
// Patch2D / Patch3D (pylops 2.x, HStack of Restriction.H over BlockDiag of Diagonal(taper) * Op), on the window
// geometry of sliding.cuh.
//
// Windows [nw0][nw1][nw2][len0][len1][len2][n_inner], data [n0][n1][nt][n_inner] (n_inner 2 for the (re, im) pairs of
// complex data); the taper is b2_sliding's table (TableTaper, nw2 = 1, len2 = nt) or b2_patch's per-axis tables
// (AxisTaper).
//   forward (fold):    d[a][b][s][k] = sum over i0 of (sum over i1 of (sum over i2 of tap[w][j0][j1][j2] * win[w]
//                      [j0][j1][j2][k])) over the windows that hold (a, b, s), j the window-local index, every sum
//                      ascending; 0 where no window holds it
//   adjoint (unfold):  win[w][j0][j1][j2][k] = tap[w][j0][j1][j2] * d[i0 step0 + j0][i1 step1 + j1][i2 step2 + j2][k]
// One thread per output value, so no atomics and no workspace: one launch per call, the same bits on every run.
#include "sliding.cuh"

namespace {

constexpr int SL_THREADS = 256;
constexpr unsigned SL_MAX_BLOCKS = 1u << 16;

template <typename T, typename Tap>
__global__ void __launch_bounds__(SL_THREADS)
fold_kernel(const T* __restrict__ win, T* __restrict__ d, long long total, long long ni, Windows g, Tap tap) {
  constexpr bool TW = Tap::time_windows;
  const long long inner = g.len2 * ni, section = g.nt * ni;   // values per window trace, per section trace
  for (long long i = (long long)blockIdx.x * SL_THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * SL_THREADS) {
    const long long tr = i / section, r = i - tr * section;   // r = s * ni + k
    const long long a = tr / g.n1, b = tr - a * g.n1;
    long long f0, l0, f1, l1, f2 = 0, l2 = 0, s = 0;
    covering(a, g.nw0, g.len0, g.step0, f0, l0);
    covering(b, g.nw1, g.len1, g.step1, f1, l1);
    if (TW) {
      s = r / ni;
      covering(s, g.nw2, g.len2, g.step2, f2, l2);
    }
    T out = T(0);
    for (long long i0 = f0; i0 <= l0; ++i0) {
      T part = T(0);
      for (long long i1 = f1; i1 <= l1; ++i1) {
        const long long j0 = a - i0 * g.step0, j1 = b - i1 * g.step1;
        const T* wt = win + (((i0 * g.nw1 + i1) * g.nw2 * g.len0 + j0) * g.len1 + j1) * inner + r;
        T q = T(0);
        for (long long i2 = f2; i2 <= l2; ++i2) {   // !TW: i2 = 0 only
          const T x = __ldg(wt + i2 * (g.len0 * g.len1 * inner - g.step2 * ni));
          const T y = tap.on() ? mul_rn(tap.sample(g, tap.trace(g, i0, i1, j0, j1), i2, s - i2 * g.step2), x) : x;
          if (TW)
            q = add_rn(q, y);
          else
            part = add_rn(part, y);
        }
        if (TW) part = add_rn(part, q);
      }
      out = add_rn(out, part);
    }
    d[i] = out;
  }
}

template <typename T, typename Tap>
__global__ void __launch_bounds__(SL_THREADS)
unfold_kernel(const T* __restrict__ d, T* __restrict__ win, long long total, long long ni, Windows g, Tap tap) {
  constexpr bool TW = Tap::time_windows;
  const long long inner = g.len2 * ni;
  for (long long i = (long long)blockIdx.x * SL_THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * SL_THREADS) {
    const long long t = i / inner, r = i - t * inner;        // t = (w * len0 + j0) * len1 + j1, r = j2 * ni + k
    const long long q = t / g.len1, j1 = t - q * g.len1;
    const long long w = q / g.len0, j0 = q - w * g.len0;
    const long long i01 = TW ? w / g.nw2 : w, i2 = w - i01 * g.nw2;
    const long long i0 = i01 / g.nw1, i1 = i01 - i0 * g.nw1;
    const T x = __ldg(d + (((i0 * g.step0 + j0) * g.n1 + i1 * g.step1 + j1) * g.nt + i2 * g.step2) * ni + r);
    win[i] = tap.on() ? mul_rn(tap.sample(g, tap.trace(g, i0, i1, j0, j1), i2, TW ? r / ni : 0), x) : x;
  }
}

template <typename MakeTap>
int overlap_add(const void* x, void* y, const Windows& g, long long ni, MakeTap make_tap, int adjoint, int dtype,
                void* stream) {
  const long long total = (adjoint ? g.nw0 * g.nw1 * g.nw2 * g.len0 * g.len1 * g.len2 : g.n0 * g.n1 * g.nt) * ni;
  const long long want = (total + SL_THREADS - 1) / SL_THREADS;
  const unsigned blocks = (unsigned)(want < (long long)SL_MAX_BLOCKS ? want : SL_MAX_BLOCKS);
  return b2_dispatch_real(dtype, [&](auto t) -> int {
    using T = decltype(t);
    const T* xs = static_cast<const T*>(x);
    T* ys = static_cast<T*>(y);
    const auto tap = make_tap(t);
    if (adjoint)
      unfold_kernel<<<blocks, SL_THREADS, 0, (cudaStream_t)stream>>>(xs, ys, total, ni, g, tap);
    else
      fold_kernel<<<blocks, SL_THREADS, 0, (cudaStream_t)stream>>>(xs, ys, total, ni, g, tap);
    B2_LAUNCH_CHECK();
    return B2_OK;
  });
}

}  // namespace

extern "C" int b2_sliding(b2_ctx* ctx, const void* x, void* y, size_t n0, size_t n1, size_t nt, size_t n_inner,
                          size_t nwins0, size_t nwins1, size_t nwin0, size_t nwin1, size_t step0, size_t step1,
                          const void* tap, int adjoint, int dtype, void* stream) {
  if (!ctx || !x || !y || x == y) return B2_ERR_ARG;
  Windows g;
  if (!make_windows(n0, n1, nt, n_inner, nwins0, nwins1, 1, nwin0, nwin1, nt, step0, step1, 1, g)) return B2_ERR_ARG;
  return overlap_add(x, y, g, (long long)n_inner,
                     [&](auto t) { return TableTaper<decltype(t)>{static_cast<const decltype(t)*>(tap)}; }, adjoint,
                     dtype, stream);
}

extern "C" int b2_patch(b2_ctx* ctx, const void* x, void* y, size_t n0, size_t n1, size_t nt, size_t n_inner,
                        size_t nwins0, size_t nwins1, size_t nwins2, size_t nwin0, size_t nwin1, size_t nwin2,
                        size_t step0, size_t step1, size_t step2, const double* tap0, const double* tap1,
                        const double* tap2, int adjoint, int dtype, void* stream) {
  if (!ctx || !x || !y || x == y) return B2_ERR_ARG;
  Windows g;
  if (!make_windows(n0, n1, nt, n_inner, nwins0, nwins1, nwins2, nwin0, nwin1, nwin2, step0, step1, step2, g))
    return B2_ERR_ARG;
  return overlap_add(x, y, g, (long long)n_inner, [&](auto t) { return AxisTaper<decltype(t)>{tap0, tap1, tap2}; },
                     adjoint, dtype, stream);
}
