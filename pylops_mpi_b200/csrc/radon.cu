// Rank-local Radon transform: pylops.signalprocessing.Radon2D / Radon3D (pylops 2.x, Spread with per-sample index
// and weight tables), on unitless axes the host prepares (local.py: h in samples of dh, p in samples of dt per dh).
//
// Model [npy][npx][nt] (2-D: npy = 1), data [nhy][nhx][nt] (2-D: nhy = 1), each sample n_inner (1, or 2 for the
// (re, im) pairs of complex data) values.  For model sample (p, t0) and trace h, in float64:
//   cx = term(hx, px), cy = term(hy, py)                 linear p*h, parabolic p*(h*h), hyperbolic (h/p)*(h/p)
//   tdec = (t0 + cx) + cy                                linear, parabolic
//   tdec = sqrt((t0*t0 + cx) + cy)                       hyperbolic (t0*t0 formed in 64-bit integers)
// In 2-D (hy = py = NULL) the y term is never formed: a zero y axis would turn every hyperbolic tdec into NaN.
//   interp:  used iff 0 <= tdec < nt - 1; it = trunc(tdec), d = tdec - it;
//            forward y[h][it] += (1 - d) x[p][t0], y[h][it + 1] += d x[p][t0]; adjoint the exact transpose
//   !interp: used iff 0 <= tdec < nt; forward y[h][trunc(tdec)] += x[p][t0]
// Every operation is an explicit round-to-nearest intrinsic, so no fma contraction can move a pair, and both
// directions evaluate the same expression: they are exact transposes of each other.  Sums are float64 and rounded
// once to the data's type.
//
// Adjoint (stacking, a gather): one thread per model sample, lanes on consecutive t0 of one model trace, so that for
// the linear and parabolic kinds (one shift per trace) a warp reads consecutive samples.  The CTA puts the cx terms
// of a tile of traces in shared memory (one divide per term, not per sample); each thread then walks the traces in
// (hy, hx) order and adds x[it] (1 - d) + x[it + 1] d per trace in registers.
//
// Forward (spreading, computed as a gather): tdec is non-decreasing in t0 for every kind (each rounded operation is
// monotone), so the t0 that reach data sample s form one contiguous range: tdec in [s - 1, s + 1) with interp (the
// second tap of [s - 1, s), the first of [s, s + 1)), [s, s + 1) without.  One thread per data sample, lanes on
// consecutive s of one trace, walks the model traces in (py, px) order; for each it estimates the first t0 of the
// range from the inverse curve, corrects the estimate with the exact expression, and adds the taps of t0 ascending
// until tdec leaves the range.  A model trace whose terms are not finite (hyperbolic p = 0) gives NaN or inf for
// every t0 and is skipped, as the mask drops all its pairs.  No atomics and no workspace: one launch per apply, the
// same bits on every run.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int RD_THREADS = 256;

template <typename T>
__device__ __forceinline__ double ld(const T* p) { return (double)__ldg(p); }

// the offset term of one (trace, model trace) pair on one axis
template <int KIND>
__device__ __forceinline__ double term(double h, double p) {
  if (KIND == B2_RADON_LINEAR) return __dmul_rn(p, h);
  if (KIND == B2_RADON_PARABOLIC) return __dmul_rn(p, __dmul_rn(h, h));
  const double q = __ddiv_rn(h, p);
  return __dmul_rn(q, q);
}

// tdec of model sample t0 given the terms of its pair
template <int KIND>
__device__ __forceinline__ double curve(long long t0, double cx, double cy, bool three) {
  double v = __dadd_rn(KIND == B2_RADON_HYPERBOLIC ? (double)(t0 * t0) : (double)t0, cx);
  if (three) v = __dadd_rn(v, cy);
  return KIND == B2_RADON_HYPERBOLIC ? __dsqrt_rn(v) : v;
}

// an estimate of the first t0 with tdec >= lo, for a finite total term c, in [0, nt]; callers correct it exactly
template <int KIND>
__device__ __forceinline__ long long first_guess(double lo, double c, long long nt) {
  double e;
  if (KIND == B2_RADON_HYPERBOLIC) {
    const double r = lo * lo - c;
    e = r > 0.0 ? ceil(sqrt(r)) : 0.0;
  } else {
    e = ceil(lo - c);
  }
  return (long long)fmin(fmax(e, 0.0), (double)nt);
}

// ---- adjoint: stacking ------------------------------------------------------------------------------------------
// CTA b covers t0 in [(b % ntb) * RD_THREADS, +RD_THREADS) of model trace b / ntb (= ipy * npx + ipx)
template <typename T, int C, int KIND>
__global__ void __launch_bounds__(RD_THREADS)
radon_stack_kernel(const T* __restrict__ x, T* __restrict__ y, long long nt, long long ntb, long long nhy,
                   long long nhx, long long npx, const double* __restrict__ hy, const double* __restrict__ hx,
                   const double* __restrict__ py, const double* __restrict__ px, bool interp) {
  __shared__ double sx[RD_THREADS];
  const long long iq = blockIdx.x / ntb;
  const long long t0 = (blockIdx.x - iq * ntb) * RD_THREADS + threadIdx.x;
  const long long ipy = iq / npx, ipx = iq - ipy * npx;
  const bool three = hy != nullptr, live = t0 < nt;
  const double pxv = __ldg(px + ipx);
  const double lim = (double)(interp ? nt - 1 : nt);
  double acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0.0;
  for (long long jy = 0; jy < nhy; ++jy) {
    const double cy = three ? term<KIND>(__ldg(hy + jy), __ldg(py + ipy)) : 0.0;
    for (long long j0 = 0; j0 < nhx; j0 += RD_THREADS) {
      const int nk = (int)min((long long)RD_THREADS, nhx - j0);
      __syncthreads();
      if ((int)threadIdx.x < nk) sx[threadIdx.x] = term<KIND>(__ldg(hx + j0 + threadIdx.x), pxv);
      __syncthreads();
      if (!live) continue;
      const T* xt = x + (size_t)(jy * nhx + j0) * nt * C;
      for (int k = 0; k < nk; ++k, xt += (size_t)nt * C) {
        const double v = curve<KIND>(t0, sx[k], cy, three);
        if (!(v >= 0.0 && v < lim)) continue;
        const long long it = (long long)v;
        const T* xs = xt + (size_t)it * C;
        if (interp) {
          const double d = __dadd_rn(v, -(double)it), w0 = __dadd_rn(1.0, -d);
#pragma unroll
          for (int c = 0; c < C; ++c)
            acc[c] = __dadd_rn(acc[c], __dadd_rn(__dmul_rn(ld(xs + c), w0), __dmul_rn(ld(xs + C + c), d)));
        } else {
#pragma unroll
          for (int c = 0; c < C; ++c) acc[c] = __dadd_rn(acc[c], ld(xs + c));
        }
      }
    }
  }
  if (live) {
#pragma unroll
    for (int c = 0; c < C; ++c) y[((size_t)iq * nt + t0) * C + c] = (T)acc[c];
  }
}

// ---- forward: spreading ------------------------------------------------------------------------------------------
// CTA b covers samples s in [(b % ntb) * RD_THREADS, +RD_THREADS) of trace b / ntb (= jy * nhx + jx)
template <typename T, int C, int KIND>
__global__ void __launch_bounds__(RD_THREADS)
radon_spread_kernel(const T* __restrict__ x, T* __restrict__ y, long long nt, long long ntb, long long nhx,
                    long long npy, long long npx, const double* __restrict__ hy, const double* __restrict__ hx,
                    const double* __restrict__ py, const double* __restrict__ px, bool interp) {
  __shared__ double sx[RD_THREADS];
  const long long jh = blockIdx.x / ntb;
  const long long s = (blockIdx.x - jh * ntb) * RD_THREADS + threadIdx.x;
  const long long jy = jh / nhx, jx = jh - jy * nhx;
  const bool three = hy != nullptr, live = s < nt;
  const double hxv = __ldg(hx + jx);
  // tdec range of the model samples that reach s; with interp the mask tdec < nt - 1 caps it
  const double lo = (double)(interp && s > 0 ? s - 1 : s);
  const double hi = interp ? fmin((double)(s + 1), (double)(nt - 1)) : (double)(s + 1);
  double acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 0.0;
  for (long long ipy = 0; ipy < npy; ++ipy) {
    const double cy = three ? term<KIND>(__ldg(hy + jy), __ldg(py + ipy)) : 0.0;
    for (long long i0 = 0; i0 < npx; i0 += RD_THREADS) {
      const int nk = (int)min((long long)RD_THREADS, npx - i0);
      __syncthreads();
      if ((int)threadIdx.x < nk) sx[threadIdx.x] = term<KIND>(hxv, __ldg(px + i0 + threadIdx.x));
      __syncthreads();
      if (!live) continue;
      const T* xm = x + (size_t)(ipy * npx + i0) * nt * C;
      for (int k = 0; k < nk; ++k, xm += (size_t)nt * C) {
        const double cx = sx[k];
        const double c = three ? cx + cy : cx;
        if (!isfinite(c)) continue;
        long long t = first_guess<KIND>(lo, c, nt);
        while (t > 0 && curve<KIND>(t - 1, cx, cy, three) >= lo) --t;
        for (; t < nt; ++t) {
          const double v = curve<KIND>(t, cx, cy, three);
          if (!(v >= lo)) continue;             // below the range: the estimate was short
          if (!(v < hi)) break;
          const T* xs = xm + (size_t)t * C;
          if (interp) {
            const long long it = (long long)v;
            const double d = __dadd_rn(v, -(double)it);
            const double w = it == s ? __dadd_rn(1.0, -d) : d;
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = __dadd_rn(acc[c], __dmul_rn(ld(xs + c), w));
          } else {
#pragma unroll
            for (int c = 0; c < C; ++c) acc[c] = __dadd_rn(acc[c], ld(xs + c));
          }
        }
      }
    }
  }
  if (live) {
#pragma unroll
    for (int c = 0; c < C; ++c) y[((size_t)jh * nt + s) * C + c] = (T)acc[c];
  }
}

template <typename T, int C, int KIND>
int launch(const void* xv, void* yv, size_t nt, size_t nhy, size_t nhx, size_t npy, size_t npx, const double* hy,
           const double* hx, const double* py, const double* px, bool interp, bool adjoint, size_t blocks,
           cudaStream_t st) {
  const T* x = static_cast<const T*>(xv);
  T* y = static_cast<T*>(yv);
  const long long ntb = (long long)((nt + RD_THREADS - 1) / RD_THREADS);
  if (adjoint)
    radon_stack_kernel<T, C, KIND><<<(unsigned)blocks, RD_THREADS, 0, st>>>(
        x, y, (long long)nt, ntb, (long long)nhy, (long long)nhx, (long long)npx, hy, hx, py, px, interp);
  else
    radon_spread_kernel<T, C, KIND><<<(unsigned)blocks, RD_THREADS, 0, st>>>(
        x, y, (long long)nt, ntb, (long long)nhx, (long long)npy, (long long)npx, hy, hx, py, px, interp);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

template <typename T, int C>
int launch_kind(int kind, const void* x, void* y, size_t nt, size_t nhy, size_t nhx, size_t npy, size_t npx,
                const double* hy, const double* hx, const double* py, const double* px, bool interp, bool adjoint,
                size_t blocks, cudaStream_t st) {
  switch (kind) {
    case B2_RADON_LINEAR:
      return launch<T, C, B2_RADON_LINEAR>(x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp, adjoint, blocks, st);
    case B2_RADON_PARABOLIC:
      return launch<T, C, B2_RADON_PARABOLIC>(x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp, adjoint, blocks,
                                              st);
    default:
      return launch<T, C, B2_RADON_HYPERBOLIC>(x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp, adjoint, blocks,
                                               st);
  }
}

}  // namespace

extern "C" int b2_radon(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t nhy, size_t nhx,
                        size_t npy, size_t npx, const double* hy, const double* hx, const double* py,
                        const double* px, int kind, int interp, int adjoint, int dtype, void* stream) {
  if (!ctx || !x || !y || x == y || !hx || !px || (hy == nullptr) != (py == nullptr)) return B2_ERR_ARG;
  if (!hy && (nhy != 1 || npy != 1)) return B2_ERR_ARG;
  const size_t axis_max = (size_t)1 << 31;
  for (size_t n : {nt, nhy, nhx, npy, npx})
    if (n == 0 || n >= axis_max) return B2_ERR_ARG;
  if (n_inner != 1 && n_inner != 2) return B2_ERR_ARG;
  if (kind != B2_RADON_LINEAR && kind != B2_RADON_PARABOLIC && kind != B2_RADON_HYPERBOLIC) return B2_ERR_ARG;
  // one CTA per RD_THREADS samples of each output trace, in one grid
  const size_t ntb = (nt + RD_THREADS - 1) / RD_THREADS;
  const size_t traces = adjoint ? npy * npx : nhy * nhx;
  if (traces > 0x7fffffffULL / ntb) return B2_ERR_ARG;
  const size_t blocks = traces * ntb;
  return b2_dispatch_real(dtype, [&](auto t) {
    using T = decltype(t);
    auto go = n_inner == 1 ? launch_kind<T, 1> : launch_kind<T, 2>;
    return go(kind, x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp != 0, adjoint != 0, blocks,
              (cudaStream_t)stream);
  });
}
