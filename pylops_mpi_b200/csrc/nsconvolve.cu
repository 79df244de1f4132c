// Rank-local NON-STATIONARY 1-D convolution along one axis of a C-ordered [n_outer][n_axis][n_inner] block: the role
// of pylops.signalprocessing.NonStationaryConvolve1D, and with a derivative stage of the 2-D wavelet branch of
// pylops.avo.poststack.PoststackLinearModelling, inside MPIBlockDiag.
//
// Filter bank hs [nfilt][nh] at the regularly spaced samples oh, oh + dh, ...; model sample j uses
//   v = (j - oh) / dh (float64), l = floor(v), w = v - l
//   h_j = hs[0] (l < 0), hs[nfilt-1] (l >= nfilt-1), hs[l] (w == 0), else T(1-w) * hs[l] + T(w) * hs[l+1]
// (two rounded products and one rounded add, never an fma: pylops' _interpolate_h under NumPy's promotion).
//   forward  y[i] = sum_j h_j[hc + i - j] x[j]       (a scatter: sample j spreads its own filter)
//   adjoint  x[j] = sum_i h_j[hc + i - j] y[i]       (the exact transpose)
// Samples outside [0, n_axis) are zero.  Both sums run in ascending j (forward) / i (adjoint), so repeated applies
// give identical bits; every term is one fma.
//
// A CTA covers RB = 64 rows along the axis x 32 columns: lanes of a warp run across the columns (the middle axis:
// columns of n_inner; the innermost axis: 32 lines, staged transposed) and share the axis rows, so every tap a
// thread reads is a broadcast.  Per chunk of kc taps the CTA interpolates the taps its rows need ONCE into shared
// memory, laid out per output row: A[q][t] is the q-th term of output row t,
//   forward  A[q][t] = h_{jb+t+q}[khi-1-q]  on the window w[m] = x[jb + m],  jb = i0 + hc - khi + 1
//   adjoint  A[q][t] = h_{j0+t}[k0+q]       on the window w[m] = y[ib + m],  ib = j0 - hc + k0
// so that both directions are the same correlation acc[t] += A[q][t] w[t + q] in ascending q, and a thread's RT
// consecutive rows read their taps A[q][t0 .. t0+RT) as one aligned vector (no diagonal reads: no bank conflicts).
// Forward chunks run from the highest taps down (ascending j), adjoint chunks from the lowest up (ascending i).
//
// Compile-time derivative stage DS, as in convolve.cu (PoststackLinearModelling = C D, D the first derivative):
//   DS_FWD  the loader stages x one row wider on each side and turns it into d = D x in shared memory
//   DS_ADJ  the tile computes e = C^T y on its RB rows and stores the inner RB - 2 rows of D^T e
// with the stencil's arithmetic (fd_axis.cuh), so the fused operator equals the two-launch chain bit for bit.
#include "common.cuh"
#include "fd_axis.cuh"

namespace {

constexpr int NS_LANES = 32, NS_GROUPS = 8, NS_THREADS = NS_LANES * NS_GROUPS;
constexpr int NS_RT = 8;                       // rows per thread
constexpr int NS_RB = NS_GROUPS * NS_RT;       // rows per CTA
constexpr int NS_WS = NS_LANES + 1;            // shared row stride of the windows (transposed staging is conflict-free)
constexpr int NS_KC = 48;                      // taps per chunk (a multiple of NS_RT)
constexpr int LAY_MID = 0, LAY_LINE = 1;       // columns of n_inner / whole lines (n_inner == 1)

struct NsParams {
  long long n;         // axis length
  long long ncols;     // columns: n_inner (LAY_MID) or lines (LAY_LINE)
  long long sa, sc;    // element strides along the axis and across columns
  long long plane;     // elements per outer index (LAY_MID; blockIdx.y)
  long long ctiles, rtiles;
  long long oh, dh;
  int nfilt, nh, hc, kc, nchunks;
};

// per-row interpolation: h_j[k] = hs[lo][k] (hi < 0) or a * hs[lo][k] + b * hs[hi][k]
template <typename T>
struct RowW { int lo, hi; T a, b; };

template <typename T>
__device__ __forceinline__ RowW<T> row_weights(long long j, const NsParams& p) {
  RowW<T> r;
  const double v = (double)(j - p.oh) / (double)p.dh;
  const double fl = floor(v);
  r.hi = -1;
  r.a = T(1);
  r.b = T(0);
  if (fl < 0.0) {
    r.lo = 0;
  } else if (fl >= (double)(p.nfilt - 1)) {
    r.lo = p.nfilt - 1;
  } else {
    r.lo = (int)fl;
    const double w = v - fl;
    if (w != 0.0) {
      r.hi = r.lo + 1;
      r.a = T(1.0 - w);
      r.b = T(w);
    }
  }
  return r;
}

__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

template <typename T>
__device__ __forceinline__ T tap_of(const RowW<T>& r, const T* __restrict__ hs, int k, int nh) {
  if (k < 0 || k >= nh) return T(0);                  // the chunk's padding taps
  const T h0 = __ldg(hs + (size_t)r.lo * nh + k);
  if (r.hi < 0) return h0;
  return add_rn(mul_rn(r.a, h0), mul_rn(r.b, __ldg(hs + (size_t)r.hi * nh + k)));
}

template <typename T, int LAY, int DS>
__global__ void __launch_bounds__(NS_THREADS, 2)
nsconv_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ hs, const NsParams p, const int adjoint,
              const int kind) {
  constexpr int XH = DS == DS_FWD ? 1 : 0;   // extra staged rows on each side (x for d = D x)
  constexpr int EH = DS == DS_ADJ ? 1 : 0;   // e rows computed on each side of the stored rows
  constexpr int RO = NS_RB - 2 * EH;         // rows stored per tile
  extern __shared__ __align__(64) unsigned char ns_smem[];
  const int rows = NS_RB + p.kc;             // window rows (the rolling register window reads one past RB + kc - 1)
  T* A = reinterpret_cast<T*>(ns_smem);                          // [kc][RB] taps
  RowW<T>* rw = reinterpret_cast<RowW<T>*>(A + (size_t)p.kc * NS_RB);   // [rows] interpolation weights
  T* w = reinterpret_cast<T*>(rw + rows);                        // [rows][WS] window (d for DS_FWD)
  T* xs = DS == DS_FWD ? w + (size_t)rows * NS_WS : w;           // DS_FWD: [rows + 2][WS] rows of x

  long long ct, rt;
  if constexpr (LAY == LAY_LINE) { rt = blockIdx.x % p.rtiles; ct = blockIdx.x / p.rtiles; }
  else { ct = blockIdx.x % p.ctiles; rt = blockIdx.x / p.ctiles; }
  const long long r0 = rt * RO - EH;                             // first row computed
  if constexpr (LAY == LAY_MID) {
    x += (size_t)blockIdx.y * p.plane;
    y += (size_t)blockIdx.y * p.plane;
  }
  const long long c0 = ct * NS_LANES;
  const int ncol = (int)min((long long)NS_LANES, p.ncols - c0);
  const int tid = threadIdx.x, lane = tid % NS_LANES, grp = tid / NS_LANES, t0 = grp * NS_RT;
  const T* xc = x + c0 * p.sc;

  T acc[NS_RT];
#pragma unroll
  for (int r = 0; r < NS_RT; ++r) acc[r] = T(0);

  for (int ch = 0; ch < p.nchunks; ++ch) {
    // forward: taps [khi - kc, khi), highest chunk first; adjoint: taps [k0, k0 + kc), lowest first
    const int k0 = adjoint ? ch * p.kc : p.nh - (ch + 1) * p.kc;
    const long long b = adjoint ? r0 - p.hc + k0 : r0 + p.hc - (k0 + p.kc) + 1;   // axis row of w[0]
    __syncthreads();                                               // the previous chunk's readers are done
    const int nw = adjoint ? NS_RB : rows;                         // rows whose filters the chunk needs
    for (int m = tid; m < nw; m += NS_THREADS) rw[m] = row_weights<T>(adjoint ? r0 + m : b + m, p);
    const int xrows = rows + 2 * XH;
    const long long bs = b - XH;
    if constexpr (LAY == LAY_LINE) {                               // consecutive threads read along a line
      for (int e = tid; e < xrows * NS_LANES; e += NS_THREADS) {
        const int l = e / xrows, m = e - l * xrows;
        const long long j = bs + m;
        xs[m * NS_WS + l] = (l < ncol && j >= 0 && j < p.n) ? __ldg(xc + (size_t)l * p.sc + j) : T(0);
      }
    } else {                                                       // consecutive threads read across columns
      for (int e = tid; e < xrows * NS_LANES; e += NS_THREADS) {
        const int m = e / NS_LANES, l = e - m * NS_LANES;
        const long long j = bs + m;
        xs[m * NS_WS + l] = (l < ncol && j >= 0 && j < p.n) ? __ldg(xc + (size_t)j * p.sa + l) : T(0);
      }
    }
    __syncthreads();
    for (int e = tid; e < p.kc * NS_RB; e += NS_THREADS) {
      const int q = e / NS_RB, t = e - q * NS_RB;
      A[e] = adjoint ? tap_of(rw[t], hs, k0 + q, p.nh) : tap_of(rw[t + q], hs, k0 + p.kc - 1 - q, p.nh);
    }
    if constexpr (DS == DS_FWD) {
      for (int e = tid; e < rows * NS_LANES; e += NS_THREADS) {
        const int m = e / NS_LANES, l = e - m * NS_LANES;
        const T* s = xs + m * NS_WS + l;                           // x[b + m - 1], x[b + m], x[b + m + 1]
        w[m * NS_WS + l] = fd_fwd(s[0], s[NS_WS], s[2 * NS_WS], b + m, p.n, kind);
      }
    }
    __syncthreads();
    using VA = VecN<T, NS_RT>;
    const T* wl = w + t0 * NS_WS + lane;
    T lo[NS_RT];
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) lo[r] = wl[r * NS_WS];
    for (int q0 = 0; q0 < p.kc; q0 += NS_RT) {
      T hi[NS_RT];
#pragma unroll
      for (int r = 0; r < NS_RT; ++r) hi[r] = wl[(q0 + NS_RT + r) * NS_WS];
#pragma unroll
      for (int qq = 0; qq < NS_RT; ++qq) {
        const VA a = *reinterpret_cast<const VA*>(A + (q0 + qq) * NS_RB + t0);
#pragma unroll
        for (int r = 0; r < NS_RT; ++r) acc[r] = fma(a.v[r], r + qq < NS_RT ? lo[r + qq] : hi[r + qq - NS_RT], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < NS_RT; ++r) lo[r] = hi[r];
    }
  }
  if constexpr (DS == DS_ADJ) {
    __syncthreads();                                               // the window is free: row t holds e[r0 + t]
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) w[(t0 + r) * NS_WS + lane] = acc[r];
    __syncthreads();
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) {
      const int t = t0 + r;
      if (t == 0 || t == NS_RB - 1) continue;
      acc[r] = fd_adj(w[(t - 1) * NS_WS + lane], w[t * NS_WS + lane], w[(t + 1) * NS_WS + lane], r0 + t, p.n, kind);
    }
  }
  if constexpr (LAY == LAY_MID) {
    if (lane >= ncol) return;
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) {
      const int t = t0 + r;
      const long long i = r0 + t;
      if (i >= p.n) break;
      if (EH && (t == 0 || t == NS_RB - 1)) continue;
      __stcs(y + (size_t)i * p.sa + c0 + lane, acc[r]);
    }
  } else {
    // lines: stage the tile transposed, then store along the lines
    __syncthreads();
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) w[(t0 + r) * NS_WS + lane] = acc[r];
    __syncthreads();
    const long long i0 = r0 + EH;
    const int nr = (int)min((long long)RO, p.n - i0);
    for (int e = tid; e < nr * NS_LANES; e += NS_THREADS) {
      const int l = e / nr, t = e - l * nr;
      if (l < ncol) __stcs(y + (size_t)(c0 + l) * p.sc + i0 + t, w[(t + EH) * NS_WS + l]);
    }
  }
}

template <typename T, int LAY, int DS>
int launch_lay(const T* x, T* y, const T* hs, size_t n_outer, size_t n, size_t ni, int nfilt, int nh, int hc,
               long long oh, long long dh, int adjoint, int kind, cudaStream_t st) {
  constexpr int RO = DS == DS_ADJ ? NS_RB - 2 : NS_RB;
  NsParams p;
  p.n = (long long)n;
  p.kc = (nh < NS_KC ? nh + NS_RT - 1 : NS_KC) / NS_RT * NS_RT;
  p.nchunks = (nh + p.kc - 1) / p.kc;
  p.oh = oh;
  p.dh = dh;
  p.nfilt = nfilt;
  p.nh = nh;
  p.hc = hc;
  p.rtiles = (long long)((n + RO - 1) / RO);
  const size_t rows = (size_t)NS_RB + p.kc;
  const size_t smem = (size_t)p.kc * NS_RB * sizeof(T) + rows * sizeof(RowW<T>) +
                      (rows + (DS == DS_FWD ? rows + 2 : 0)) * NS_WS * sizeof(T);
  const int rc = b2_allow_smem<nsconv_kernel<T, LAY, DS>>(smem);
  if (rc != B2_OK) return rc;
  if constexpr (LAY == LAY_LINE) {
    // columns are whole lines: launch groups of lines so that the grid stays within 2^31 - 1 blocks
    p.sa = 1;
    p.sc = (long long)n;
    p.plane = 0;
    return b2_launch_groups(n_outer, (size_t)(0x7fffffffLL / p.rtiles) * NS_LANES, [&](size_t first, size_t cnt) {
      p.ncols = (long long)cnt;
      p.ctiles = (long long)((cnt + NS_LANES - 1) / NS_LANES);
      nsconv_kernel<T, LAY, DS><<<(unsigned)(p.ctiles * p.rtiles), NS_THREADS, smem, st>>>(
          x + first * n, y + first * n, hs, p, adjoint, kind);
    });
  } else {
    p.sa = (long long)ni;
    p.sc = 1;
    p.plane = (long long)(n * ni);
    p.ncols = (long long)ni;
    p.ctiles = (long long)((ni + NS_LANES - 1) / NS_LANES);
    const long long nblk = p.ctiles * p.rtiles;
    if (nblk > 0x7fffffffLL) return B2_ERR_ARG;
    return b2_launch_groups(n_outer, B2_GRID_Y_MAX, [&](size_t first, size_t cnt) {
      const size_t o = first * n * ni;
      nsconv_kernel<T, LAY, DS><<<dim3((unsigned)nblk, (unsigned)cnt), NS_THREADS, smem, st>>>(x + o, y + o, hs, p,
                                                                                             adjoint, kind);
    });
  }
}

template <typename T, int DS>
int launch_ns(const void* x, void* y, const void* hs, size_t n_outer, size_t n, size_t ni, int nfilt, int nh, int hc,
              long long oh, long long dh, int adjoint, int kind, cudaStream_t st) {
  const T* xt = static_cast<const T*>(x);
  T* yt = static_cast<T*>(y);
  const T* h = static_cast<const T*>(hs);
  if (ni == 1)
    return launch_lay<T, LAY_LINE, DS>(xt, yt, h, n_outer, n, ni, nfilt, nh, hc, oh, dh, adjoint, kind, st);
  return launch_lay<T, LAY_MID, DS>(xt, yt, h, n_outer, n, ni, nfilt, nh, hc, oh, dh, adjoint, kind, st);
}

// Both entry points.  Unlike convolve.cu's, an empty block is B2_ERR_ARG; a bad kind wins over a bad dtype
int ns_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner, const void* hs,
            int nfilt, int nh, int hc, long long oh, long long dh, bool fused, int kind, int adjoint, int dtype,
            void* stream) {
  if (!ctx || !x || !y || !hs || x == y) return B2_ERR_ARG;
  if (n_outer == 0 || n_axis == 0 || n_inner == 0) return B2_ERR_ARG;
  if (nfilt < 1 || nh < 1 || hc < 0 || hc >= nh || dh < 1) return B2_ERR_ARG;
  if (fused && kind != B2_FD_CENTERED && kind != B2_FD_FORWARD) return B2_ERR_ARG;
  return ds_dispatch(dtype, fused, adjoint, [&](auto t, auto ds) {
    return launch_ns<decltype(t), decltype(ds)::value>(x, y, hs, n_outer, n_axis, n_inner, nfilt, nh, hc, oh, dh,
                                                       adjoint ? 1 : 0, kind, (cudaStream_t)stream);
  });
}

}  // namespace

extern "C" int b2_nsconvolve_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                                  const void* hs, int nfilt, int nh, int hc, long long oh, long long dh, int adjoint,
                                  int dtype, void* stream) {
  return ns_axis(ctx, x, y, n_outer, n_axis, n_inner, hs, nfilt, nh, hc, oh, dh, false, 0, adjoint, dtype, stream);
}

extern "C" int b2_nspoststack_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis,
                                   size_t n_inner, const void* hs, int nfilt, int nh, int hc, long long oh,
                                   long long dh, int kind, int adjoint, int dtype, void* stream) {
  return ns_axis(ctx, x, y, n_outer, n_axis, n_inner, hs, nfilt, nh, hc, oh, dh, true, kind, adjoint, dtype, stream);
}
