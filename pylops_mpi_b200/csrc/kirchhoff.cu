// Rank-local Kirchhoff demigration, spreading / stacking stage: pylops.waveeqprocessing.Kirchhoff (pylops 2.x,
// mode="analytic", 2-D or 3-D, dynamic=False) without its wavelet convolution, which runs as b2_convolve_axis.  This is
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
//
// Chunks (b2_kirchhoff_chunk): the same two kernels over the image points [i0, i0 + nc) with that chunk's tables.
// The forward adds into the traces instead of zeroing them when asked to; with i0 a multiple of 32 its warp steps
// cover the same 32 points as in one call over [0, ni), so chunks applied in ascending order give the same bits.
//
// Tables (b2_kirchhoff_tables): pylops' analytic traveltime, one thread per image point looping over the points
// (sources or receivers), with NumPy's operations in NumPy's order and explicit round-to-nearest intrinsics:
//   2-D  sqrt((x - px)*(x - px) + (z - pz)*(z - pz)) / vel
//   3-D  sqrt(((x - px)*(x - px) + (z - pz)*(z - pz)) + (y - py)*(y - py)) / vel
// (NumPy's `**2` is x*x; its sqrt and divide are correctly rounded), so they equal the host NumPy tables bit for bit.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int KH_ADJ_THREADS = 128;
constexpr int KH_ADJ_UNROLL = 4;
constexpr int KH_FWD_WARPS = 4;                           // warps (traces) per CTA, forward
// dynamic shared memory of the forward's trace buffers: the default 48 KB per CTA less the static group scratch
constexpr size_t KH_FWD_SMEM = 48 * 1024 - 2 * KH_FWD_WARPS * 32 * sizeof(double);
constexpr int KH_TAB_THREADS = 256;
constexpr unsigned KH_TAB_ROWS = 64;                     // table builder: grid rows, each takes every 64th point

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
// accumulate: the trace starts from y's values instead of zero.
template <typename T, bool SMEM>
__global__ void __launch_bounds__(KH_FWD_WARPS * 32)
kirchhoff_spread_kernel(const T* __restrict__ x, T* __restrict__ y, const double* __restrict__ ts,
                        const double* __restrict__ tr, long long ni, int ns, int nr, long long nt, double dt,
                        bool accumulate) {
  extern __shared__ __align__(16) unsigned char kh_smem[];
  __shared__ double sc0[KH_FWD_WARPS][32], sc1[KH_FWD_WARPS][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long g = (long long)blockIdx.x * KH_FWD_WARPS + warp;   // receiver-major trace number
  if (g >= (long long)ns * nr) return;
  const int r = (int)(g / ns), s = (int)(g - (long long)r * ns);
  T* yt = y + ((size_t)s * nr + r) * nt;
  T* acc = SMEM ? reinterpret_cast<T*>(kh_smem) + (size_t)warp * nt : yt;
  if (SMEM || !accumulate)
    for (long long t = lane; t < nt; t += 32) acc[t] = accumulate ? yt[t] : T(0);
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

// ---- traveltime tables -------------------------------------------------------------------------------------------
// One thread per image point ii = i0 + j (its grid coordinates are loaded once); the grid's y dimension splits the
// n points, so each thread writes every gridDim.y-th row of table[n][nc], coalesced along j.
__global__ void __launch_bounds__(KH_TAB_THREADS)
kirchhoff_table_kernel(const double* __restrict__ ay, const double* __restrict__ ax, const double* __restrict__ az,
                       long long nx, long long nz, const double* __restrict__ pts, long long n, double vel,
                       long long i0, long long nc, double* __restrict__ table) {
  const long long j = (long long)blockIdx.x * KH_TAB_THREADS + threadIdx.x;
  if (j >= nc) return;
  const long long ii = i0 + j, rest = ii / nz;
  const bool three = ay != nullptr;
  const double gx = __ldg(ax + rest % nx), gz = __ldg(az + ii - rest * nz);
  const double gy = three ? __ldg(ay + rest / nx) : 0.0;
  const double* px = pts + (three ? n : 0);          // rows (y,) x, z
  const double* pz = px + n;
  for (long long p = blockIdx.y; p < n; p += gridDim.y) {
    const double dx = __dsub_rn(gx, __ldg(px + p)), dz = __dsub_rn(gz, __ldg(pz + p));
    double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dz, dz));
    if (three) {
      const double dy = __dsub_rn(gy, __ldg(pts + p));
      d2 = __dadd_rn(d2, __dmul_rn(dy, dy));
    }
    table[(size_t)p * nc + j] = __ddiv_rn(__dsqrt_rn(d2), vel);
  }
}

template <typename T>
int launch(const void* xv, void* yv, const double* ts, const double* tr, size_t ni, int ns, int nr, size_t nt,
           double dt, int adjoint, bool accumulate, cudaStream_t st) {
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
        x, y, ts, tr, (long long)ni, ns, nr, (long long)nt, dt, accumulate);
  else
    kirchhoff_spread_kernel<T, false><<<(unsigned)blocks, KH_FWD_WARPS * 32, 0, st>>>(
        x, y, ts, tr, (long long)ni, ns, nr, (long long)nt, dt, accumulate);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

// the checks b2_kirchhoff and b2_kirchhoff_chunk share
int check_args(b2_ctx* ctx, const void* x, void* y, const double* ts, const double* tr, size_t ni, size_t ns,
               size_t nr, size_t nt, double dt) {
  if (!ctx || !x || !y || !ts || !tr || x == y) return B2_ERR_ARG;
  if (ni == 0 || ns == 0 || nr == 0 || nt < 1) return B2_ERR_ARG;
  if (ns > 0x7fffffffULL || nr > 0x7fffffffULL) return B2_ERR_ARG;
  if (!(dt > 0.0) || !isfinite(dt)) return B2_ERR_ARG;
  return B2_OK;
}

// image points [i0, i0 + nc): the image side (x forward, y adjoint) starts at i0, the tables hold the chunk only;
// B2_ERR_DTYPE for a dtype other than F32 / F64, after every other check of the entry points
int apply(const void* x, void* y, const double* ts, const double* tr, size_t i0, size_t nc, size_t ns, size_t nr,
          size_t nt, double dt, int adjoint, bool accumulate, int dtype, cudaStream_t st) {
  return b2_dispatch_real(dtype, [&](auto t) {
    using T = decltype(t);
    const T* xt = static_cast<const T*>(x) + (adjoint ? 0 : i0);
    T* yt = static_cast<T*>(y) + (adjoint ? i0 : 0);
    return launch<T>(xt, yt, ts, tr, nc, (int)ns, (int)nr, nt, dt, adjoint, accumulate, st);
  });
}

}  // namespace

extern "C" int b2_kirchhoff(b2_ctx* ctx, const void* x, void* y, const double* trav_srcs, const double* trav_recs,
                            size_t ni, size_t ns, size_t nr, size_t nt, double dt, int adjoint, int dtype,
                            void* stream) {
  const int rc = check_args(ctx, x, y, trav_srcs, trav_recs, ni, ns, nr, nt, dt);
  if (rc != B2_OK) return rc;
  return apply(x, y, trav_srcs, trav_recs, 0, ni, ns, nr, nt, dt, adjoint, false, dtype, (cudaStream_t)stream);
}

extern "C" int b2_kirchhoff_chunk(b2_ctx* ctx, const void* x, void* y, const double* trav_srcs,
                                  const double* trav_recs, size_t ni, size_t i0, size_t nc, size_t ns, size_t nr,
                                  size_t nt, double dt, int adjoint, int accumulate, int dtype, void* stream) {
  const int rc = check_args(ctx, x, y, trav_srcs, trav_recs, ni, ns, nr, nt, dt);
  if (rc != B2_OK) return rc;
  if (nc == 0 || i0 % 32 != 0 || i0 >= ni || nc > ni - i0) return B2_ERR_ARG;
  if (accumulate != 0 && (accumulate != 1 || adjoint)) return B2_ERR_ARG;
  return apply(x, y, trav_srcs, trav_recs, i0, nc, ns, nr, nt, dt, adjoint, accumulate != 0, dtype,
               (cudaStream_t)stream);
}

extern "C" int b2_kirchhoff_tables(b2_ctx* ctx, const double* y, const double* x, const double* z, size_t ny,
                                   size_t nx, size_t nz, const double* pts, size_t n, double vel, size_t i0,
                                   size_t nc, double* table, void* stream) {
  if (!ctx || !x || !z || !pts || !table) return B2_ERR_ARG;
  if (nx == 0 || nz == 0 || n == 0 || nc == 0 || (y && ny == 0)) return B2_ERR_ARG;
  const size_t nyy = y ? ny : 1;
  if (nx > SIZE_MAX / nz || nyy > SIZE_MAX / (nx * nz)) return B2_ERR_ARG;
  const size_t ni = nyy * nx * nz;
  if (i0 >= ni || nc > ni - i0) return B2_ERR_ARG;
  const size_t bx = (nc + KH_TAB_THREADS - 1) / KH_TAB_THREADS;
  if (bx > 0x7fffffffULL) return B2_ERR_ARG;
  const dim3 grid((unsigned)bx, (unsigned)(n < KH_TAB_ROWS ? n : KH_TAB_ROWS));
  kirchhoff_table_kernel<<<grid, KH_TAB_THREADS, 0, (cudaStream_t)stream>>>(
      y, x, z, (long long)nx, (long long)nz, pts, (long long)n, vel, (long long)i0, (long long)nc, table);
  B2_LAUNCH_CHECK();
  return B2_OK;
}
