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
//
// Windows (b2_radon_windows: pylops.signalprocessing.Sliding2D / Sliding3D over Radon2D / Radon3D; b2_radon_patches:
// Patch2D / Patch3D, on the window geometry of sliding.cuh).  The same two kernels, compiled a second time with WIN
// and the taper source: the section [n0][n1][ns] holds windows of nhy x nhx traces and nt samples (b2_radon_windows:
// nt = ns, one window along the samples), each with its own model block [npy][npx][nt] on window-local time and the
// window-local offsets hy, hx.  Forward: one thread per section sample; for each window that holds it (i2 inside i1
// inside i0, all ascending) it forms that window's value at the window-local sample exactly as above (a float64 sum
// rounded once to T), multiplies it by the window's taper in T and adds it in T in b2_sliding's / b2_patch's order.
// The windows along the samples differ between the threads of a CTA, so with them each thread walks its own windows
// and forms the offset terms itself: no CTA barrier couples warps that hold different windows.  Adjoint: one thread per model sample of window w, reading tap * d
// rounded to T at the window-local sample plus the window's first sample, where the one-gather kernel reads d.  Both
// equal b2_radon per window plus b2_sliding / b2_patch bit for bit.
#include <math.h>

#include "sliding.cuh"

namespace {

constexpr int RD_THREADS = 256;

template <typename T>
__device__ __forceinline__ double ld(const T* p) { return (double)__ldg(p); }
// a data value as the windowed stack reads it: tap * d rounded to T when tapered
template <typename T>
__device__ __forceinline__ double ldt(const T* p, T tap, bool tapered) {
  return tapered ? (double)mul_rn(tap, __ldg(p)) : ld(p);
}

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
// CTA b covers t0 in [(b % ntb) * RD_THREADS, +RD_THREADS) of model trace b / ntb (= ipy * npx + ipx; WIN: of window
// w's block, (w * npy + ipy) * npx + ipx, whose traces are the section traces of window w from its first sample, each
// value tap * d in T)
template <typename T, int C, int KIND, bool WIN, typename Tap>
__device__ __forceinline__ void stack(const T* __restrict__ x, T* __restrict__ y, long long nt, long long ntb,
                                      long long nhy, long long nhx, long long npy, long long npx,
                                      const double* __restrict__ hy, const double* __restrict__ hx,
                                      const double* __restrict__ py, const double* __restrict__ px, bool interp,
                                      const Windows& win, const Tap& tap) {
  __shared__ double sx[RD_THREADS];
  const long long iq = blockIdx.x / ntb;
  const long long t0 = (blockIdx.x - iq * ntb) * RD_THREADS + threadIdx.x;
  const long long w = WIN ? iq / (npy * npx) : 0, ip = iq - w * npy * npx;
  const long long ipy = ip / npx, ipx = ip - ipy * npx;
  const bool three = hy != nullptr, live = t0 < nt, tapered = WIN && tap.on();
  const long long i01 = WIN && Tap::time_windows ? w / win.nw2 : w, i2 = w - i01 * win.nw2;
  const long long i0 = WIN ? i01 / win.nw1 : 0, i1 = i01 - i0 * win.nw1;
  const long long a0 = i0 * win.step0, b0 = i1 * win.step1, o2 = i2 * win.step2;   // WIN: the window's origin
  const long long ns = WIN ? win.nt : nt;                                          // samples per data trace
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
      const T* xt = x + ((size_t)(WIN ? (a0 + jy) * win.n1 + b0 + j0 : jy * nhx + j0) * ns + o2) * C;
      for (int k = 0; k < nk; ++k, xt += (size_t)ns * C) {
        const double v = curve<KIND>(t0, sx[k], cy, three);
        if (!(v >= 0.0 && v < lim)) continue;
        const long long it = (long long)v;
        const T* xs = xt + (size_t)it * C;
        const auto tt = tapered ? tap.trace(win, i0, i1, jy, j0 + k) : 1;
        const T tv = tapered ? tap.sample(win, tt, i2, it) : T(1);
        if (interp) {
          const double d = __dadd_rn(v, -(double)it), w0 = __dadd_rn(1.0, -d);
          const T tv1 = tapered ? tap.sample(win, tt, i2, it + 1) : T(1);
#pragma unroll
          for (int c = 0; c < C; ++c)
            acc[c] = __dadd_rn(acc[c], __dadd_rn(__dmul_rn(ldt(xs + c, tv, tapered), w0),
                                                 __dmul_rn(ldt(xs + C + c, tv1, tapered), d)));
        } else {
#pragma unroll
          for (int c = 0; c < C; ++c) acc[c] = __dadd_rn(acc[c], ldt(xs + c, tv, tapered));
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
// the tdec range [lo, hi) of the model samples that reach window-local sample s; with interp the mask tdec < nt - 1
// caps it
__device__ __forceinline__ double lo_of(long long s, bool interp) { return (double)(interp && s > 0 ? s - 1 : s); }
__device__ __forceinline__ double hi_of(long long s, long long nt, bool interp) {
  return interp ? fmin((double)(s + 1), (double)(nt - 1)) : (double)(s + 1);
}

// CTA b covers samples s in [(b % ntb) * RD_THREADS, +RD_THREADS) of trace b / ntb (= jy * nhx + jx; WIN: of section
// trace a * n1 + b, which sums the tapered values of the windows that hold it, each from that window's model block)
template <typename T, int C, int KIND, bool WIN, typename Tap>
__device__ __forceinline__ void spread(const T* __restrict__ x, T* __restrict__ y, long long nt, long long ntb,
                                       long long nhy, long long nhx, long long npy, long long npx,
                                       const double* __restrict__ hy, const double* __restrict__ hx,
                                       const double* __restrict__ py, const double* __restrict__ px, bool interp,
                                       const Windows& win, const Tap& tap) {
  constexpr bool TW = WIN && Tap::time_windows;
  __shared__ double sx[RD_THREADS];
  const long long jh = blockIdx.x / ntb;
  const long long s = (blockIdx.x - jh * ntb) * RD_THREADS + threadIdx.x;
  const long long ns = WIN ? win.nt : nt;                  // samples per data trace
  const bool three = hy != nullptr, live = s < ns;
  const double lo0 = lo_of(s, interp), hi0 = hi_of(s, nt, interp);   // !TW: s is window-local
  // the windows [f0, l0] x [f1, l1] that hold the trace, and [f2, l2] along the samples that hold s (none past the
  // section); without WIN the one gather
  long long a = 0, b = 0, f0 = 0, l0 = 0, f1 = 0, l1 = 0, f2 = 0, l2 = 0;
  if (WIN) {
    a = jh / win.n1;
    b = jh - a * win.n1;
    covering(a, win.nw0, win.len0, win.step0, f0, l0);
    covering(b, win.nw1, win.len1, win.step1, f1, l1);
  }
  if (TW) {
    covering(s, win.nw2, win.len2, win.step2, f2, l2);
    if (!live) l2 = f2 - 1;
  }
  T out[C];
#pragma unroll
  for (int c = 0; c < C; ++c) out[c] = T(0);
  for (long long i0 = f0; i0 <= l0; ++i0) {
    T part[C];
#pragma unroll
    for (int c = 0; c < C; ++c) part[c] = T(0);
    for (long long i1 = f1; i1 <= l1; ++i1) {
      const long long jy = WIN ? a - i0 * win.step0 : jh / nhx;
      const long long jx = WIN ? b - i1 * win.step1 : jh - jy * nhx;
      const double hxv = __ldg(hx + jx);
      T q[C];
#pragma unroll
      for (int c = 0; c < C; ++c) q[c] = T(0);
      for (long long i2 = f2; i2 <= l2; ++i2) {      // !TW: i2 = 0 only
      const long long w = (i0 * win.nw1 + i1) * win.nw2 + i2;
      const T* xw = WIN ? x + (size_t)w * npy * npx * nt * C : x;
      const bool in = live;
      const long long sl = TW ? s - i2 * win.step2 : s;   // the window-local sample
      const double lo = TW ? lo_of(sl, interp) : lo0, hi = TW ? hi_of(sl, nt, interp) : hi0;
      double acc[C];
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] = 0.0;
      for (long long ipy = 0; ipy < npy; ++ipy) {
        const double cy = three ? term<KIND>(__ldg(hy + jy), __ldg(py + ipy)) : 0.0;
        for (long long i0p = 0; i0p < npx; i0p += RD_THREADS) {
          const int nk = (int)min((long long)RD_THREADS, npx - i0p);
          if (!TW) {
            __syncthreads();
            if ((int)threadIdx.x < nk) sx[threadIdx.x] = term<KIND>(hxv, __ldg(px + i0p + threadIdx.x));
            __syncthreads();
          }
          if (!in) continue;
          const T* xm = xw + (size_t)(ipy * npx + i0p) * nt * C;
          for (int k = 0; k < nk; ++k, xm += (size_t)nt * C) {
            const double cx = TW ? term<KIND>(hxv, __ldg(px + i0p + k)) : sx[k];
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
                const double wt = it == sl ? __dadd_rn(1.0, -d) : d;
#pragma unroll
                for (int c = 0; c < C; ++c) acc[c] = __dadd_rn(acc[c], __dmul_rn(ld(xs + c), wt));
              } else {
#pragma unroll
                for (int c = 0; c < C; ++c) acc[c] = __dadd_rn(acc[c], ld(xs + c));
              }
            }
          }
        }
      }
      if (WIN && in) {
        const T tv = tap.on() ? tap.sample(win, tap.trace(win, i0, i1, jy, jx), i2, sl) : T(1);
#pragma unroll
        for (int c = 0; c < C; ++c) {
          const T v = tap.on() ? mul_rn(tv, (T)acc[c]) : (T)acc[c];
          if (TW)
            q[c] = add_rn(q[c], v);
          else
            part[c] = add_rn(part[c], v);
        }
      } else if (!WIN) {
#pragma unroll
        for (int c = 0; c < C; ++c) out[c] = (T)acc[c];
      }
      }
      if (TW) {
#pragma unroll
        for (int c = 0; c < C; ++c) part[c] = add_rn(part[c], q[c]);
      }
    }
    if (WIN) {
#pragma unroll
      for (int c = 0; c < C; ++c) out[c] = add_rn(out[c], part[c]);
    }
  }
  if (live) {
#pragma unroll
    for (int c = 0; c < C; ++c) y[((size_t)jh * ns + s) * C + c] = out[c];
  }
}

#define RADON_KERNEL_ARGS                                                                                          \
  const T *__restrict__ x, T *__restrict__ y, long long nt, long long ntb, long long nhy, long long nhx, long long npy, \
      long long npx, const double *__restrict__ hy, const double *__restrict__ hx, const double *__restrict__ py,      \
      const double *__restrict__ px, bool interp, Windows win, Tap tap
#define RADON_BODY_ARGS x, y, nt, ntb, nhy, nhx, npy, npx, hy, hx, py, px, interp, win, tap

// the one-gather kernels of b2_radon (Tap unused) and the windowed ones of b2_radon_windows (TableTaper) and
// b2_radon_patches (AxisTaper); the windowed spreading kernel and the patches' stacking kernel, whose window loops and
// per-sample tapers keep more values live, are allowed the registers they need (no spills) by a minimum of one CTA
// per SM
template <typename T, int C, int KIND, typename Tap>
__global__ void __launch_bounds__(RD_THREADS) radon_stack_kernel(RADON_KERNEL_ARGS) {
  stack<T, C, KIND, false>(RADON_BODY_ARGS);
}
template <typename T, int C, int KIND, typename Tap>
__global__ void __launch_bounds__(RD_THREADS) radon_spread_kernel(RADON_KERNEL_ARGS) {
  spread<T, C, KIND, false>(RADON_BODY_ARGS);
}
template <typename T, int C, int KIND, typename Tap>
__global__ void __launch_bounds__(RD_THREADS) radon_stack_windows_kernel(RADON_KERNEL_ARGS) {
  stack<T, C, KIND, true>(RADON_BODY_ARGS);
}
template <typename T, int C, int KIND, typename Tap>
__global__ void __launch_bounds__(RD_THREADS, 1) radon_stack_patches_kernel(RADON_KERNEL_ARGS) {
  stack<T, C, KIND, true>(RADON_BODY_ARGS);
}
template <typename T, int C, int KIND, typename Tap>
__global__ void __launch_bounds__(RD_THREADS, 1) radon_spread_windows_kernel(RADON_KERNEL_ARGS) {
  spread<T, C, KIND, true>(RADON_BODY_ARGS);
}

// WIN: the windows of win, with taper tap; else the one gather (win and tap unused).  nt is a window's samples;
// the forward's CTAs cover the section's win.nt samples of each trace
template <typename T, int C, int KIND, bool WIN, typename Tap>
int launch(const void* xv, void* yv, size_t nt, size_t nhy, size_t nhx, size_t npy, size_t npx, const double* hy,
           const double* hx, const double* py, const double* px, bool interp, bool adjoint, size_t blocks,
           const Windows& win, const Tap& tap, cudaStream_t st) {
  const T* x = static_cast<const T*>(xv);
  T* y = static_cast<T*>(yv);
  const size_t ns = WIN && !adjoint ? (size_t)win.nt : nt;
  const long long ntb = (long long)((ns + RD_THREADS - 1) / RD_THREADS);
  auto kernel = [&] {
    if constexpr (WIN && Tap::time_windows)
      return adjoint ? radon_stack_patches_kernel<T, C, KIND, Tap> : radon_spread_windows_kernel<T, C, KIND, Tap>;
    else if constexpr (WIN)
      return adjoint ? radon_stack_windows_kernel<T, C, KIND, Tap> : radon_spread_windows_kernel<T, C, KIND, Tap>;
    else
      return adjoint ? radon_stack_kernel<T, C, KIND, Tap> : radon_spread_kernel<T, C, KIND, Tap>;
  }();
  kernel<<<(unsigned)blocks, RD_THREADS, 0, st>>>(x, y, (long long)nt, ntb, (long long)nhy, (long long)nhx,
                                                  (long long)npy, (long long)npx, hy, hx, py, px, interp, win, tap);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

template <typename T, int C, bool WIN, typename Tap>
int launch_kind(int kind, const void* x, void* y, size_t nt, size_t nhy, size_t nhx, size_t npy, size_t npx,
                const double* hy, const double* hx, const double* py, const double* px, bool interp, bool adjoint,
                size_t blocks, const Windows& win, const Tap& tap, cudaStream_t st) {
  switch (kind) {
    case B2_RADON_LINEAR:
      return launch<T, C, B2_RADON_LINEAR, WIN>(x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp, adjoint, blocks,
                                                win, tap, st);
    case B2_RADON_PARABOLIC:
      return launch<T, C, B2_RADON_PARABOLIC, WIN>(x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp, adjoint,
                                                   blocks, win, tap, st);
    default:
      return launch<T, C, B2_RADON_HYPERBOLIC, WIN>(x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp, adjoint,
                                                    blocks, win, tap, st);
  }
}

// the windowed launch of b2_radon_windows and b2_radon_patches on window geometry win (a window's samples win.len2),
// with the taper make_tap(T()) makes: one CTA per RD_THREADS samples of each output trace (adjoint: every window's
// model traces), in one grid
template <typename MakeTap>
int launch_windows(const void* x, void* y, size_t n_inner, size_t nhy, size_t nhx, size_t npy, size_t npx,
                   const double* hy, const double* hx, const double* py, const double* px, int kind, int interp,
                   const Windows& win, MakeTap make_tap, int adjoint, int dtype, void* stream) {
  const size_t nt = (size_t)win.len2, ns = adjoint ? nt : (size_t)win.nt;
  const size_t ntb = (ns + RD_THREADS - 1) / RD_THREADS;
  const size_t mtr = npy * npx, nw = (size_t)(win.nw0 * win.nw1 * win.nw2), ntr = (size_t)(win.n0 * win.n1);
  if (adjoint && (nw > 0x7fffffffULL / mtr || nw * mtr > 0x7fffffffULL / ntb)) return B2_ERR_ARG;
  if (!adjoint && ntr > 0x7fffffffULL / ntb) return B2_ERR_ARG;
  const size_t blocks = (adjoint ? nw * mtr : ntr) * ntb;
  return b2_dispatch_real(dtype, [&](auto t) {
    using T = decltype(t);
    const auto tap = make_tap(t);
    auto go = n_inner == 1 ? launch_kind<T, 1, true, decltype(tap)> : launch_kind<T, 2, true, decltype(tap)>;
    return go(kind, x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp != 0, adjoint != 0, blocks, win, tap,
              (cudaStream_t)stream);
  });
}

// the checks b2_radon, b2_radon_windows and b2_radon_patches share
bool radon_args(b2_ctx* ctx, const void* x, const void* y, size_t nt, size_t n_inner, size_t nhy, size_t nhx,
                size_t npy, size_t npx, const double* hy, const double* hx, const double* py, const double* px,
                int kind) {
  if (!ctx || !x || !y || x == y || !hx || !px || (hy == nullptr) != (py == nullptr)) return false;
  if (!hy && (nhy != 1 || npy != 1)) return false;
  const size_t axis_max = (size_t)1 << 31;
  for (size_t n : {nt, nhy, nhx, npy, npx})
    if (n == 0 || n >= axis_max) return false;
  if (n_inner != 1 && n_inner != 2) return false;
  return kind == B2_RADON_LINEAR || kind == B2_RADON_PARABOLIC || kind == B2_RADON_HYPERBOLIC;
}

}  // namespace

extern "C" int b2_radon(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t nhy, size_t nhx,
                        size_t npy, size_t npx, const double* hy, const double* hx, const double* py,
                        const double* px, int kind, int interp, int adjoint, int dtype, void* stream) {
  if (!radon_args(ctx, x, y, nt, n_inner, nhy, nhx, npy, npx, hy, hx, py, px, kind)) return B2_ERR_ARG;
  // one CTA per RD_THREADS samples of each output trace, in one grid
  const size_t ntb = (nt + RD_THREADS - 1) / RD_THREADS;
  const size_t traces = adjoint ? npy * npx : nhy * nhx;
  if (traces > 0x7fffffffULL / ntb) return B2_ERR_ARG;
  const size_t blocks = traces * ntb;
  const Windows one{};
  return b2_dispatch_real(dtype, [&](auto t) {
    using T = decltype(t);
    const TableTaper<T> none{nullptr};
    auto go = n_inner == 1 ? launch_kind<T, 1, false, TableTaper<T>> : launch_kind<T, 2, false, TableTaper<T>>;
    return go(kind, x, y, nt, nhy, nhx, npy, npx, hy, hx, py, px, interp != 0, adjoint != 0, blocks, one, none,
              (cudaStream_t)stream);
  });
}

extern "C" int b2_radon_windows(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t n0, size_t n1,
                                size_t nhy, size_t nhx, size_t npy, size_t npx, const double* hy, const double* hx,
                                const double* py, const double* px, int kind, int interp, size_t nwins0,
                                size_t nwins1, size_t step0, size_t step1, const void* tap, int adjoint, int dtype,
                                void* stream) {
  if (!radon_args(ctx, x, y, nt, n_inner, nhy, nhx, npy, npx, hy, hx, py, px, kind)) return B2_ERR_ARG;
  Windows win;
  if (!make_windows(n0, n1, nt, n_inner, nwins0, nwins1, 1, nhy, nhx, nt, step0, step1, 1, win)) return B2_ERR_ARG;
  return launch_windows(x, y, n_inner, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, win,
                        [&](auto t) { return TableTaper<decltype(t)>{static_cast<const decltype(t)*>(tap)}; }, adjoint,
                        dtype, stream);
}

extern "C" int b2_radon_patches(b2_ctx* ctx, const void* x, void* y, size_t nt, size_t n_inner, size_t n0, size_t n1,
                                size_t ns, size_t nhy, size_t nhx, size_t npy, size_t npx, const double* hy,
                                const double* hx, const double* py, const double* px, int kind, int interp,
                                size_t nwins0, size_t nwins1, size_t nwins2, size_t step0, size_t step1, size_t step2,
                                const double* tap0, const double* tap1, const double* tap2, int adjoint, int dtype,
                                void* stream) {
  if (!radon_args(ctx, x, y, nt, n_inner, nhy, nhx, npy, npx, hy, hx, py, px, kind)) return B2_ERR_ARG;
  Windows win;
  if (!make_windows(n0, n1, ns, n_inner, nwins0, nwins1, nwins2, nhy, nhx, nt, step0, step1, step2, win))
    return B2_ERR_ARG;
  return launch_windows(x, y, n_inner, nhy, nhx, npy, npx, hy, hx, py, px, kind, interp, win,
                        [&](auto t) { return AxisTaper<decltype(t)>{tap0, tap1, tap2}; }, adjoint, dtype, stream);
}
