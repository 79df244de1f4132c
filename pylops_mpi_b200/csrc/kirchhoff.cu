// Rank-local Kirchhoff demigration, spreading / stacking stage: pylops.waveeqprocessing.Kirchhoff (pylops 2.x,
// mode="analytic", 2-D, dynamic=False) without its wavelet convolution, which runs as b2_convolve_axis.  This is
// LSM(...).Demop of tutorials/lsm.py inside MPIVStack.
//
// Image points ii in [0, ni), traces isr = isrc * nr + irec of nt samples.  For each (ii, isr) pair:
//   trav = trav_srcs[isrc][ii] + trav_recs[irec][ii]       float64 tables, one float64 add
//   q = trav / dt, it = trunc(q), d = q - it               one IEEE float64 divide (no 1/dt), as pylops computes it
//   the pair is used only when 0 <= it < nt - 1
//   forward  y[isr][it] += x[ii] (1 - d),  y[isr][it + 1] += x[ii] d
//   adjoint  y[ii] += x[isr][it] (1 - d) + x[isr][it + 1] d     (pairs in (isrc, irec) ascending order)
// The index math is float64 with explicit round-to-nearest intrinsics, so that no fma contraction can move a pair.
//
// Adjoint (stacking, a gather): one thread per image point walks the traces in pylops' order and keeps its sum in
// registers, so the float64 result equals pylops' loop bit for bit.  Receivers are processed UNROLL at a time so that
// the table and trace loads of several pairs are in flight together; the sums are still added one pair at a time.
//
// Forward (spreading, a scatter): one warp per trace; lanes take 32 consecutive image points (adjacent along z, so
// they often land on the same sample).  Lanes with equal `it` are grouped with __match_any_sync; the lowest lane of
// each group adds the group's terms in ascending lane order and writes all first taps, then, after __syncwarp, all
// second taps.  Each write phase touches distinct samples, so there are no atomics and the result does not depend on
// scheduling.  The trace is accumulated in shared memory when it fits (then written out once, coalesced), else in
// place in global memory, which the warp owns.  Warps take traces receiver-major, so that the warps running at the
// same time share one receiver table row and the source table stays in L2.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int KH_ADJ_THREADS = 128;
constexpr int KH_ADJ_UNROLL = 4;
constexpr int KH_FWD_WARPS = 4;                           // warps (traces) per CTA, forward
// dynamic shared memory of the forward's trace buffers: the default 48 KB per CTA less the static group scratch
constexpr size_t KH_FWD_SMEM = 48 * 1024 - 2 * KH_FWD_WARPS * 32 * sizeof(double);

struct Pair {
  long long it;     // first sample, valid only when ok
  double d;         // interpolation weight of the second sample
  bool ok;
};

// pylops: itrav = int(trav / dt), travd = trav / dt - itrav, used iff 0 <= itrav < nt - 1
__device__ __forceinline__ Pair pair_index(double ts, double tr, double dt, long long nt) {
  Pair p;
  const double q = __ddiv_rn(__dadd_rn(ts, tr), dt);
  // trunc(q) in [0, nt - 2]  <=>  -1 < q < nt - 1  (NaN fails both)
  p.ok = q > -1.0 && q < (double)(nt - 1);
  p.it = p.ok ? (long long)q : 0;
  p.d = __dadd_rn(q, -(double)p.it);
  return p;
}

template <typename T>
__device__ __forceinline__ double ld(const T* p) { return (double)__ldg(p); }

// ---- adjoint: stacking ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(KH_ADJ_THREADS)
kirchhoff_stack_kernel(const T* __restrict__ x, T* __restrict__ y, const double* __restrict__ ts,
                       const double* __restrict__ tr, long long ni, int ns, int nr, long long nt, double dt) {
  const long long ii = (long long)blockIdx.x * KH_ADJ_THREADS + threadIdx.x;
  if (ii >= ni) return;
  double acc = 0.0;
  for (int s = 0; s < ns; ++s) {
    const double tsi = __ldg(ts + (size_t)s * ni + ii);
    const T* xs = x + (size_t)s * nr * nt;
    int r = 0;
    for (; r + KH_ADJ_UNROLL <= nr; r += KH_ADJ_UNROLL) {
      double a[KH_ADJ_UNROLL], b[KH_ADJ_UNROLL], w[KH_ADJ_UNROLL];
      bool ok[KH_ADJ_UNROLL];
#pragma unroll
      for (int u = 0; u < KH_ADJ_UNROLL; ++u) {
        const Pair p = pair_index(tsi, __ldg(tr + (size_t)(r + u) * ni + ii), dt, nt);
        const T* xt = xs + (size_t)(r + u) * nt + p.it;
        ok[u] = p.ok;
        w[u] = p.d;
        a[u] = p.ok ? ld(xt) : 0.0;
        b[u] = p.ok ? ld(xt + 1) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < KH_ADJ_UNROLL; ++u)
        if (ok[u]) acc = __dadd_rn(acc, __dadd_rn(__dmul_rn(a[u], __dadd_rn(1.0, -w[u])), __dmul_rn(b[u], w[u])));
    }
    for (; r < nr; ++r) {
      const Pair p = pair_index(tsi, __ldg(tr + (size_t)r * ni + ii), dt, nt);
      if (p.ok) {
        const T* xt = xs + (size_t)r * nt + p.it;
        acc = __dadd_rn(acc, __dadd_rn(__dmul_rn(ld(xt), __dadd_rn(1.0, -p.d)), __dmul_rn(ld(xt + 1), p.d)));
      }
    }
  }
  y[ii] = (T)acc;
}

// ---- forward: spreading -----------------------------------------------------------------------------------------
// SMEM: the trace is accumulated in a shared buffer of nt elements per warp; else directly in y.  The accumulator
// type is T: float64 traces sum in float64, float32 traces add each float64 group sum rounded to float32.
template <typename T, bool SMEM>
__global__ void __launch_bounds__(KH_FWD_WARPS * 32)
kirchhoff_spread_kernel(const T* __restrict__ x, T* __restrict__ y, const double* __restrict__ ts,
                        const double* __restrict__ tr, long long ni, int ns, int nr, long long nt, double dt) {
  extern __shared__ __align__(16) unsigned char kh_smem[];
  __shared__ double sc0[KH_FWD_WARPS][32], sc1[KH_FWD_WARPS][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long g = (long long)blockIdx.x * KH_FWD_WARPS + warp;   // receiver-major trace number
  if (g >= (long long)ns * nr) return;
  const int r = (int)(g / ns), s = (int)(g - (long long)r * ns);
  T* yt = y + ((size_t)s * nr + r) * nt;
  T* acc = SMEM ? reinterpret_cast<T*>(kh_smem) + (size_t)warp * nt : yt;
  for (long long t = lane; t < nt; t += 32) acc[t] = T(0);
  __syncwarp();
  const double* tss = ts + (size_t)s * ni;
  const double* trr = tr + (size_t)r * ni;
  const unsigned below = (1u << lane) - 1u;
  for (long long i0 = 0; i0 < ni; i0 += 32) {
    const long long ii = i0 + lane;
    Pair p;
    p.ok = false;
    p.it = 0;
    p.d = 0.0;
    double xv = 0.0;
    if (ii < ni) {
      p = pair_index(__ldg(tss + ii), __ldg(trr + ii), dt, nt);
      xv = ld(x + ii);
    }
    sc0[warp][lane] = __dmul_rn(xv, __dadd_rn(1.0, -p.d));
    sc1[warp][lane] = __dmul_rn(xv, p.d);
    const unsigned grp = __match_any_sync(0xffffffffu, p.ok ? p.it : -1LL);
    const bool lead = p.ok && (grp & below) == 0;
    __syncwarp();
    double s0 = 0.0, s1 = 0.0;
    if (lead) {
      for (unsigned m = grp; m; m &= m - 1) {
        const int l = __ffs(m) - 1;
        s0 = __dadd_rn(s0, sc0[warp][l]);
        s1 = __dadd_rn(s1, sc1[warp][l]);
      }
      acc[p.it] = (T)__dadd_rn((double)acc[p.it], s0);           // first taps: distinct samples
    }
    __syncwarp();
    if (lead) acc[p.it + 1] = (T)__dadd_rn((double)acc[p.it + 1], s1);   // second taps: distinct samples
    __syncwarp();
  }
  if (SMEM)
    for (long long t = lane; t < nt; t += 32) yt[t] = acc[t];
}

template <typename T>
int launch(const void* xv, void* yv, const double* ts, const double* tr, size_t ni, int ns, int nr, size_t nt,
           double dt, int adjoint, cudaStream_t st) {
  const T* x = static_cast<const T*>(xv);
  T* y = static_cast<T*>(yv);
  if (adjoint) {
    const size_t blocks = (ni + KH_ADJ_THREADS - 1) / KH_ADJ_THREADS;
    if (blocks > 0x7fffffffULL) return B2_ERR_ARG;
    kirchhoff_stack_kernel<T><<<(unsigned)blocks, KH_ADJ_THREADS, 0, st>>>(x, y, ts, tr, (long long)ni, ns, nr,
                                                                           (long long)nt, dt);
    B2_LAUNCH_CHECK();
    return B2_OK;
  }
  const size_t ntr = (size_t)ns * (size_t)nr;
  const size_t blocks = (ntr + KH_FWD_WARPS - 1) / KH_FWD_WARPS;
  if (blocks > 0x7fffffffULL) return B2_ERR_ARG;
  const size_t smem = (size_t)KH_FWD_WARPS * nt * sizeof(T);
  if (smem <= KH_FWD_SMEM)
    kirchhoff_spread_kernel<T, true><<<(unsigned)blocks, KH_FWD_WARPS * 32, smem, st>>>(
        x, y, ts, tr, (long long)ni, ns, nr, (long long)nt, dt);
  else
    kirchhoff_spread_kernel<T, false><<<(unsigned)blocks, KH_FWD_WARPS * 32, 0, st>>>(
        x, y, ts, tr, (long long)ni, ns, nr, (long long)nt, dt);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

}  // namespace

extern "C" int b2_kirchhoff(b2_ctx* ctx, const void* x, void* y, const double* trav_srcs, const double* trav_recs,
                            size_t ni, size_t ns, size_t nr, size_t nt, double dt, int adjoint, int dtype,
                            void* stream) {
  if (!ctx || !x || !y || !trav_srcs || !trav_recs || x == y) return B2_ERR_ARG;
  if (ni == 0 || ns == 0 || nr == 0 || nt < 1) return B2_ERR_ARG;
  if (ns > 0x7fffffffULL || nr > 0x7fffffffULL) return B2_ERR_ARG;
  if (!(dt > 0.0) || !isfinite(dt)) return B2_ERR_ARG;
  if (dtype != B2_F32 && dtype != B2_F64) return B2_ERR_DTYPE;
  cudaStream_t st = (cudaStream_t)stream;
  return dtype == B2_F32
             ? launch<float>(x, y, trav_srcs, trav_recs, ni, (int)ns, (int)nr, nt, dt, adjoint, st)
             : launch<double>(x, y, trav_srcs, trav_recs, ni, (int)ns, (int)nr, nt, dt, adjoint, st);
}
