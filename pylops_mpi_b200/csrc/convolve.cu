// Rank-local 1-D convolution along one axis of a C-ordered [n_outer][n_axis][n_inner] block: the role of
// pylops.signalprocessing.Convolve1D inside MPIBlockDiag (tutorials/reflectivity.py:74-76).
//
//   forward  y[i] = sum_k h[k] x[i + offset - k]      (x outside [0, n_axis) is zero)
//   adjoint  the same formula with h reversed and offset' = nh - 1 - offset (the exact transpose)
//
// Both kernels stage the input rows a tile needs in shared memory (zero-filled outside the line) together with a
// chunk of at most KC taps, stored reversed so that the inner loop is a correlation
//   y[t] += sum_q g[q] w[t + q],   g[q] = h[k0 + kc - 1 - q],   w[m] = x[t0 + offset - k0 - kc + 1 + m].
// Every thread produces R consecutive outputs from a rolling register window: each 16-byte shared-memory read
// feeds R*R (innermost) or RT*RT*V (middle axis) FMAs.  Tap chunks and taps within a chunk are summed in a fixed
// order, so repeated applies give identical bits.
//
// The same kernels also run pylops.avo.poststack.PoststackLinearModelling, C D with D the first derivative
// along the axis (FirstDerivative, edge=False, sampling=1), through a compile-time derivative stage DS:
//   DS_FWD  y = C D x: the loader stages x with one extra sample on each side and turns it into d = D x in shared
//           memory; the correlation then runs unchanged on d.
//   DS_ADJ  x = D^T C^T y: the correlation computes e = C^T y on the tile plus one neighbour on each side, and the
//           epilogue applies D^T to e from shared memory.
// d and D^T e use the stencil kernel's arithmetic (stencil.cu: non-zero taps in ascending offset order, each an fma
// into an accumulator that starts at 0), and e the same tap chunks as b2_convolve_axis, so the fused operator
// equals the two-launch chain b2_derivative_axis + b2_convolve_axis bit for bit (fd_fwd / fd_adj: fd_axis.cuh).
#include "common.cuh"
#include "fd_axis.cuh"

namespace {

constexpr int CV_THREADS = 256;
constexpr int CV_KC_LINE = 128;              // taps per chunk, innermost axis
constexpr int CV_KC_MID = 64;                // taps per chunk, middle axis
constexpr size_t CV_SMEM_BUDGET = 32 * 1024; // bytes of staged windows per CTA (packed short lines)

// ---- innermost axis (n_inner == 1) ----------------------------------------------------------------------------
// A CTA covers L lines x S outputs (S = R * ceil(n / R) capped at the tile, L = tile / S when lines are short).
struct LineParams {
  long long n;        // line length
  long long nlines;
  long long tiles;    // tiles per line
  int S, L, W, kc;    // outputs per line segment, lines per CTA, window stride (S + kc), taps per chunk
  int nh, off, adjoint;
  int vec;            // L == 1, n % R == 0 and x 16-byte aligned: every line starts on a 16-byte boundary
};

template <typename T>
__device__ __forceinline__ T tap(const T* __restrict__ h, int k, int nh, int adjoint) {
  return k < nh ? __ldg(h + (adjoint ? nh - 1 - k : k)) : T(0);
}

// DS_FWD: the window of x, one sample wider on each side, is staged in a second buffer after the L windows and
// turned into d.  DS_ADJ: a tile's outputs only need e on [i0 - 1, i0 + S]; when a line spans several tiles
// (then L == 1) thread 0 computes e[i0 - 1] and the last thread e[i0 + S], with the same tap order as the others,
// so the 16-byte tile geometry and stores of the plain convolution are kept.
template <typename T, int DS>
__global__ void __launch_bounds__(CV_THREADS)
conv_line_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ h, const LineParams p,
                 const int kind) {
  constexpr int R = Vec16<T>::N;
  constexpr int XH = DS == DS_FWD ? 1 : 0;  // extra staged samples on each side of the window
  extern __shared__ __align__(16) unsigned char cv_smem[];
  T* g = reinterpret_cast<T*>(cv_smem);     // kc reversed taps (kc is a multiple of R: w stays 16-byte aligned)
  T* w = g + p.kc;                          // L windows of W elements
  T* xs = DS == DS_FWD ? w + p.L * p.W : w; // DS_FWD: L windows of x of W + 2 elements
  const int Ws = p.W + 2 * XH;
  const long long grp = (long long)blockIdx.x / p.tiles;
  const long long i0 = ((long long)blockIdx.x - grp * p.tiles) * p.S;
  const long long line0 = grp * p.L;
  const int nl = (int)min((long long)p.L, p.nlines - line0);
  const int lt = threadIdx.x * R;
  const int l = lt / p.S, li = lt - l * p.S;
  const bool active = l < nl;
  T acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = T(0);
  T hlo = T(0), hhi = T(0);                 // DS_ADJ: e[i0 - 1] (thread 0), e[i0 + S] (last thread)

  for (int k0 = 0; k0 < p.nh; k0 += p.kc) {
    __syncthreads();                                   // the previous chunk's readers are done
    for (int q = threadIdx.x; q < p.kc; q += CV_THREADS) g[q] = tap(h, k0 + p.kc - 1 - q, p.nh, p.adjoint);
    const long long b = i0 + p.off - k0 - p.kc + 1;    // line index of w[0]
    const long long bs = b - XH;                       // line index of xs[0]
    if (p.vec) {
      // one line per CTA, 16-byte aligned line: aligned vector loads of the R-blocks covering the window
      const T* xl = x + line0 * p.n;
      const long long a = bs >= 0 ? bs / R * R : -((-bs + R - 1) / R) * R;
      const int nv = (int)((bs + Ws - a + R - 1) / R);
      for (int v = threadIdx.x; v < nv; v += CV_THREADS) {
        const long long j0 = a + (long long)v * R;
        Vec16<T> o;
        if (j0 >= 0 && j0 + R <= p.n) o = load_vec(xl + j0);
        else
#pragma unroll
          for (int e = 0; e < R; ++e) o.v[e] = (j0 + e >= 0 && j0 + e < p.n) ? __ldg(xl + j0 + e) : T(0);
#pragma unroll
        for (int e = 0; e < R; ++e) {
          const long long m = j0 + e - bs;
          if (m >= 0 && m < Ws) xs[m] = o.v[e];
        }
      }
    } else {
      const int tot = nl * Ws;
      for (int e = threadIdx.x; e < tot; e += CV_THREADS) {
        const int ll = e / Ws, m = e - ll * Ws;
        const long long j = bs + m;
        xs[e] = (j >= 0 && j < p.n) ? __ldg(x + (line0 + ll) * p.n + j) : T(0);
      }
    }
    if constexpr (DS == DS_FWD) {
      __syncthreads();
      const int tot = nl * p.W;
      for (int e = threadIdx.x; e < tot; e += CV_THREADS) {
        const int ll = e / p.W, m = e - ll * p.W;
        const T* s = xs + ll * Ws + m;                 // x[b + m - 1], x[b + m], x[b + m + 1]
        w[e] = fd_fwd(s[0], s[1], s[2], b + m, p.n, kind);
      }
    }
    __syncthreads();
    if (active) {
      using VR = VecN<T, R>;
      const VR* wl = reinterpret_cast<const VR*>(w + l * p.W + li);     // W, li and kc are multiples of R
      const VR* gv = reinterpret_cast<const VR*>(g);
      VR lo = wl[0];
      for (int q = 0; q < p.kc / R; ++q) {
        const VR hi = wl[q + 1];
        const VR gq = gv[q];
#pragma unroll
        for (int qq = 0; qq < R; ++qq)
#pragma unroll
          for (int r = 0; r < R; ++r) acc[r] = fma(gq.v[qq], r + qq < R ? lo.v[r + qq] : hi.v[r + qq - R], acc[r]);
        lo = hi;
      }
    }
    if constexpr (DS == DS_ADJ) {
      if (p.tiles > 1 && threadIdx.x == 0) {           // e[i0 - 1] = sum_q g[q] w[q - 1], w[-1] = x[b - 1]
        const T* xl = x + line0 * p.n;
        hlo = fma(g[0], (b - 1 >= 0 && b - 1 < p.n) ? __ldg(xl + b - 1) : T(0), hlo);
        for (int q = 1; q < p.kc; ++q) hlo = fma(g[q], w[q - 1], hlo);
      } else if (p.tiles > 1 && threadIdx.x == CV_THREADS - 1) {   // e[i0 + S] = sum_q g[q] w[S + q]
        for (int q = 0; q < p.kc; ++q) hhi = fma(g[q], w[p.S + q], hhi);
      }
    }
  }
  if constexpr (DS == DS_ADJ) {
    __syncthreads();                                   // the window is free: it now holds e
    T* e = w + l * p.W + 1;                            // e[t] = e[i0 + t] of this thread's line, t in [-1, S]
    if (active)
#pragma unroll
      for (int r = 0; r < R; ++r) e[li + r] = acc[r];
    if (p.tiles > 1 && threadIdx.x == 0) w[0] = hlo;
    if (p.tiles > 1 && threadIdx.x == CV_THREADS - 1) w[p.S + 1] = hhi;
    __syncthreads();
    if (active)
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = fd_adj(e[li + r - 1], e[li + r], e[li + r + 1], i0 + li + r, p.n, kind);
  }
  if (!active) return;
  const long long i = i0 + li;
  T* yp = y + (line0 + l) * p.n + i;
  if (i + R <= p.n && (((uintptr_t)yp) & 15u) == 0) {
    Vec16<T> o;
#pragma unroll
    for (int r = 0; r < R; ++r) o.v[r] = acc[r];
    store_vec(yp, o);
  } else {
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (i + r < p.n) __stcs(yp + r, acc[r]);
  }
}

// ---- middle axis (n_inner > 1) --------------------------------------------------------------------------------
// CTA = 16 lanes across n_inner (V columns each) x 16 row groups of RT rows: RB = 64 output rows of COLS columns.
// The RB + kc input rows the tile needs are staged per tap chunk; consecutive row tiles overlap in L2.
constexpr int MID_LANES = 16, MID_GROUPS = 16, MID_RT = 4, MID_RB = MID_GROUPS * MID_RT;
struct MidParams {
  long long n, ni;    // axis length, inner length (elements of T)
  long long ctiles;   // column tiles
  int kc, nh, off, adjoint;
};

template <typename T, int V>
__device__ __forceinline__ VecN<T, V> ld_vec(const T* p) {
  VecN<T, V> o;
  if constexpr (V * sizeof(T) == 16) *reinterpret_cast<uint4*>(&o) = ldg_stream16(p);
  else
#pragma unroll
    for (int e = 0; e < V; ++e) o.v[e] = __ldg(p + e);
  return o;
}

template <typename T, int V, int DS>
__global__ void __launch_bounds__(MID_LANES * MID_GROUPS)
conv_mid_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ h, const MidParams p,
                const int kind) {
  constexpr int COLS = MID_LANES * V;
  constexpr int XH = DS == DS_FWD ? 1 : 0;  // extra staged rows on each side of the window
  constexpr int EH = DS == DS_ADJ ? 1 : 0;  // e rows computed on each side of the stored rows
  constexpr int RO = MID_RB - 2 * EH;       // rows stored per tile
  extern __shared__ __align__(16) unsigned char cv_smem[];
  T* g = reinterpret_cast<T*>(cv_smem);     // kc taps (kc is a multiple of MID_RT)
  VecN<T, V>* w = reinterpret_cast<VecN<T, V>*>(g + p.kc);   // (RB + kc) rows x MID_LANES vectors
  const long long ct = (long long)blockIdx.x % p.ctiles;
  const long long r0 = ((long long)blockIdx.x / p.ctiles) * RO - EH;   // first row computed
  const size_t plane = (size_t)p.n * (size_t)p.ni;
  x += (size_t)blockIdx.y * plane;
  y += (size_t)blockIdx.y * plane;
  const int lane = threadIdx.x, grp = threadIdx.y, tid = grp * MID_LANES + lane;
  const long long c = ct * COLS + (long long)lane * V;   // first column of this lane
  const bool col_ok = c < p.ni;                          // V divides ni whenever V > 1
  T acc[MID_RT][V];
#pragma unroll
  for (int r = 0; r < MID_RT; ++r)
#pragma unroll
    for (int e = 0; e < V; ++e) acc[r][e] = T(0);

  const int rows = MID_RB + p.kc;
  VecN<T, V>* xs = DS == DS_FWD ? w + rows * MID_LANES : w;   // DS_FWD: rows + 2 rows of x
  for (int k0 = 0; k0 < p.nh; k0 += p.kc) {
    __syncthreads();
    for (int q = tid; q < p.kc; q += MID_LANES * MID_GROUPS) g[q] = tap(h, k0 + p.kc - 1 - q, p.nh, p.adjoint);
    const long long b = r0 + p.off - k0 - p.kc + 1;     // axis index of staged row 0
    for (int m = grp; m < rows + 2 * XH; m += MID_GROUPS) {
      const long long j = b - XH + m;
      VecN<T, V> v;
      if (col_ok && j >= 0 && j < p.n) v = ld_vec<T, V>(x + (size_t)j * p.ni + c);
      else
#pragma unroll
        for (int e = 0; e < V; ++e) v.v[e] = T(0);
      xs[m * MID_LANES + lane] = v;
    }
    if constexpr (DS == DS_FWD) {
      __syncthreads();
      for (int m = grp; m < rows; m += MID_GROUPS) {
        const VecN<T, V>* s = xs + m * MID_LANES + lane;   // rows b + m - 1, b + m, b + m + 1
        const VecN<T, V> a = s[0], o = s[MID_LANES], z = s[2 * MID_LANES];
        VecN<T, V> d;
#pragma unroll
        for (int e = 0; e < V; ++e) d.v[e] = fd_fwd(a.v[e], o.v[e], z.v[e], b + m, p.n, kind);
        w[m * MID_LANES + lane] = d;
      }
    }
    __syncthreads();
    const VecN<T, V>* wl = w + (grp * MID_RT) * MID_LANES + lane;
    VecN<T, V> lo[MID_RT];
#pragma unroll
    for (int r = 0; r < MID_RT; ++r) lo[r] = wl[r * MID_LANES];
    for (int q0 = 0; q0 < p.kc; q0 += MID_RT) {
      VecN<T, V> hi[MID_RT];
#pragma unroll
      for (int r = 0; r < MID_RT; ++r) hi[r] = wl[(q0 + MID_RT + r) * MID_LANES];
#pragma unroll
      for (int qq = 0; qq < MID_RT; ++qq) {
        const T gq = g[q0 + qq];
#pragma unroll
        for (int r = 0; r < MID_RT; ++r)
#pragma unroll
          for (int e = 0; e < V; ++e)
            acc[r][e] = fma(gq, r + qq < MID_RT ? lo[r + qq].v[e] : hi[r + qq - MID_RT].v[e], acc[r][e]);
      }
#pragma unroll
      for (int r = 0; r < MID_RT; ++r) lo[r] = hi[r];
    }
  }
  if constexpr (DS == DS_ADJ) {
    __syncthreads();                                    // the window is free: row t of it now holds e[r0 + t]
#pragma unroll
    for (int r = 0; r < MID_RT; ++r)
#pragma unroll
      for (int e = 0; e < V; ++e) w[(grp * MID_RT + r) * MID_LANES + lane].v[e] = acc[r][e];
    __syncthreads();
#pragma unroll
    for (int r = 0; r < MID_RT; ++r) {
      const int t = grp * MID_RT + r;
      if (t == 0 || t == MID_RB - 1) continue;
      const VecN<T, V> a = w[(t - 1) * MID_LANES + lane], o = w[t * MID_LANES + lane], z = w[(t + 1) * MID_LANES + lane];
#pragma unroll
      for (int e = 0; e < V; ++e) acc[r][e] = fd_adj(a.v[e], o.v[e], z.v[e], r0 + t, p.n, kind);
    }
  }
  if (!col_ok) return;
#pragma unroll
  for (int r = 0; r < MID_RT; ++r) {
    const long long i = r0 + grp * MID_RT + r;
    if (i >= p.n) break;
    if (DS == DS_ADJ && (grp * MID_RT + r == 0 || grp * MID_RT + r == MID_RB - 1)) continue;
    T* yp = y + (size_t)i * p.ni + c;
    if constexpr (V * sizeof(T) == 16) {
      store_vec(yp, *reinterpret_cast<const Vec16<T>*>(&acc[r][0]));
    } else {
#pragma unroll
      for (int e = 0; e < V; ++e) __stcs(yp + e, acc[r][e]);
    }
  }
}

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

template <typename T, int DS>
int launch_line(const T* x, T* y, const T* h, size_t n_lines, size_t n, int nh, int off, int adjoint, int kind,
                cudaStream_t st) {
  constexpr int R = Vec16<T>::N, TILE = CV_THREADS * R;
  LineParams p;
  p.kc = round_up(nh < CV_KC_LINE ? nh : CV_KC_LINE, R);
  p.S = (int)(n < (size_t)TILE ? round_up((int)n, R) : TILE);
  p.W = p.S + p.kc;
  const int per_line = DS == DS_FWD ? 2 * p.W + 2 : p.W;      // DS_FWD also stages x, W + 2 per line
  const int fit = (int)((CV_SMEM_BUDGET / sizeof(T) - p.kc) / per_line);
  p.L = TILE / p.S < fit ? TILE / p.S : fit;
  if (p.L < 1) p.L = 1;
  p.n = (long long)n;
  p.tiles = (long long)((n + p.S - 1) / p.S);
  p.nh = nh;
  p.off = off;
  p.adjoint = adjoint;
  p.vec = p.L == 1 && n % R == 0 && b2_aligned16(x);
  const size_t smem = ((size_t)p.kc + (size_t)p.L * per_line) * sizeof(T);
  const size_t max_groups = (size_t)(0x7fffffffLL / p.tiles);
  return b2_launch_groups(n_lines, (max_groups / p.L) * p.L, [&](size_t first, size_t cnt) {
    p.nlines = (long long)cnt;
    const size_t blocks = (cnt + p.L - 1) / p.L * (size_t)p.tiles;
    conv_line_kernel<T, DS><<<(unsigned)blocks, CV_THREADS, smem, st>>>(x + first * n, y + first * n, h, p, kind);
  });
}

template <typename T, int V, int DS>
int launch_mid_v(const T* x, T* y, const T* h, size_t n_outer, size_t n, size_t ni, int nh, int off, int adjoint,
                 int kind, cudaStream_t st) {
  constexpr int COLS = MID_LANES * V, RO = DS == DS_ADJ ? MID_RB - 2 : MID_RB;   // rows stored per tile
  MidParams p;
  p.kc = round_up(nh < CV_KC_MID ? nh : CV_KC_MID, MID_RT);
  p.n = (long long)n;
  p.ni = (long long)ni;
  p.ctiles = (long long)((ni + COLS - 1) / COLS);
  p.nh = nh;
  p.off = off;
  p.adjoint = adjoint;
  const long long nblk = p.ctiles * (long long)((n + RO - 1) / RO);
  if (nblk > 0x7fffffffLL) return B2_ERR_ARG;
  const size_t rows = (size_t)(MID_RB + p.kc) + (DS == DS_FWD ? MID_RB + p.kc + 2 : 0);   // DS_FWD: + rows of x
  const size_t smem = (size_t)p.kc * sizeof(T) + rows * MID_LANES * V * sizeof(T);
  const int rc = b2_allow_smem<conv_mid_kernel<T, V, DS>>(smem);   // DS_FWD with kc > 20 taps needs more than 48 KB
  if (rc != B2_OK) return rc;
  return b2_launch_groups(n_outer, B2_GRID_Y_MAX, [&](size_t first, size_t cnt) {
    const size_t o = first * n * ni;
    conv_mid_kernel<T, V, DS><<<dim3((unsigned)nblk, (unsigned)cnt), dim3(MID_LANES, MID_GROUPS), smem, st>>>(
        x + o, y + o, h, p, kind);
  });
}

template <typename T, int DS>
int launch_conv(const void* xv, void* yv, const void* hv, size_t n_outer, size_t n, size_t ni, int nh, int off,
                int adjoint, int kind, cudaStream_t st) {
  const T* x = static_cast<const T*>(xv);
  T* y = static_cast<T*>(yv);
  const T* h = static_cast<const T*>(hv);
  if (adjoint) off = nh - 1 - off;     // exact transpose: reversed taps (read in the kernel), mirrored offset
  if (ni == 1) return launch_line<T, DS>(x, y, h, n_outer, n, nh, off, adjoint, kind, st);
  constexpr int V = Vec16<T>::N;
  if (ni % V == 0 && b2_aligned16(x) && b2_aligned16(y))
    return launch_mid_v<T, V, DS>(x, y, h, n_outer, n, ni, nh, off, adjoint, kind, st);
  return launch_mid_v<T, 1, DS>(x, y, h, n_outer, n, ni, nh, off, adjoint, kind, st);
}

// Both entry points.  Callers see the order of the checks: a bad kind wins over a bad dtype, and an empty block is
// B2_OK without a launch (and before x and y are looked at)
int conv_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner, const void* h,
              int nh, int offset, bool fused, int kind, int adjoint, int dtype, void* stream) {
  if (!ctx || nh < 1 || offset < 0 || offset > nh - 1 || !h) return B2_ERR_ARG;
  if (fused && kind != B2_FD_CENTERED && kind != B2_FD_FORWARD) return B2_ERR_ARG;
  if (dtype != B2_F32 && dtype != B2_F64) return B2_ERR_DTYPE;
  if (n_outer == 0 || n_axis == 0 || n_inner == 0) return B2_OK;
  if (!x || !y || x == y) return B2_ERR_ARG;
  return ds_dispatch(dtype, fused, adjoint, [&](auto t, auto ds) {
    return launch_conv<decltype(t), decltype(ds)::value>(x, y, h, n_outer, n_axis, n_inner, nh, offset,
                                                         adjoint ? 1 : 0, kind, (cudaStream_t)stream);
  });
}

}  // namespace

extern "C" int b2_convolve_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                                const void* h, int nh, int offset, int adjoint, int dtype, void* stream) {
  return conv_axis(ctx, x, y, n_outer, n_axis, n_inner, h, nh, offset, false, 0, adjoint, dtype, stream);
}

extern "C" int b2_poststack_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                                 const void* h, int nh, int offset, int kind, int adjoint, int dtype, void* stream) {
  return conv_axis(ctx, x, y, n_outer, n_axis, n_inner, h, nh, offset, true, kind, adjoint, dtype, stream);
}
