// Rank-local NON-STATIONARY 3-D convolution of a C-ordered [nx][ny][nz][n_inner] volume: the role of
// pylops.signalprocessing.NonStationaryConvolve3D inside MPIBlockDiag (n_inner = 2: complex data as (re, im) pairs).
//
// Filter bank hs [nfx][nfy][nfz][nhx][nhy][nhz] at the points (ohx + a dhx, ohy + b dhy, ohz + e dhz), centre
// (hcx, hcy, hcz) = (nhx / 2, nhy / 2, nhz / 2).  Point j = (jx, jy, jz) uses h_j = sum_(a,b,e) W_abe[j] hs[a][b][e],
// with separable trilinear weights
//   W_abe[j] = T((wz_e(jz) * wy_b(jy)) * wx_a(jx))   (the float64 product in this order, rounded once to the type T)
// and per axis  v = (j - oh) / dh (float64), l = floor(v), w = v - l:  weight 1 on filter 0 (l < 0) or on filter nf - 1
// (l >= nf - 1), else 1 - w on l and w on l + 1.
//   forward  y[i] = sum_j h_j[hc + i - j] x[j]       (a scatter: point j spreads its own filter)
//   adjoint  x[j] = sum_i h_j[hc + i - j] y[i]       (the exact transpose)
// Points outside the volume are zero.
//
// Scheme: the trilinear decomposition, as nsconvolve2d.cu's bilinear one.  Since h_j is linear in the bank,
//   forward  y = sum_c h_c * (W_c . x)               adjoint  x = sum_c W_c . (h_c (x) y)
// (c = (a, b, e) over the bank).  W_c is non-zero only on the support S_c of filter c, so a CTA of TX x 32 x 64
// outputs runs, for each filter whose support reaches it, one STATIONARY correlation restricted to the taps that can
// meet the support.  The 3-D correlation is a sum over x tap planes of 2-D correlations: the CTA stages one (y, z)
// input plane at a time in shared memory (double-buffered, one barrier per plane), and each staged plane feeds every
// one of the TX output planes it reaches (tap plane = input plane - output plane), so a window value loaded into
// registers serves up to TX tap planes (correlate_plane, ns_core.cuh).  Within a plane the tile is nsconvolve2d.cu's
// with its own chunk size: lanes of a warp run along y (one output row each, every tap a broadcast), a thread's RT = 8
// consecutive z outputs slide a register window along z, and the window row stride is odd.  Taps go in chunks of KCX x KCY x KCZ: any filter size fits the fixed shared
// memory, filters larger than the volume included.
//   forward  the window holds u_c = W_c . x (zero off S_c) and the taps are reversed: acc[t] += h_c[K-1-q] u_c[t + q]
//   adjoint  the window holds y, v[t] += h_c[q] y[t + q] over the whole filter, then acc[t] = fma(W_c[t], v[t], acc[t])
// Sum order: filters in ascending (a, b, e); within a filter, tap chunks in ascending (x, y, z) order and the taps of a
// chunk in ascending (x, y, z) order (forward: of the reversed filter), one fma per term.  No atomics, no allocation:
// repeated applies give identical bits.  The sums differ from pylops' (interpolate h_j, then convolve) only in
// rounding; with exactly representable inputs both are exact.
#include "ns_core.cuh"

namespace {

constexpr int N3_TY = NS_LANES;                            // outputs per plane of a CTA: 32 (y) x 64 (z)
constexpr int N3_KCX = 16;                                 // tap planes per chunk (x)
constexpr int N3_KC = 16;                                  // taps per chunk along y and z (a multiple of NS_RT)
constexpr int N3_WR = N3_TY + N3_KC - 1;                   // window rows (y)
constexpr int N3_WC = NS_TZ + N3_KC;                       // window columns (z): the register window reads one past
constexpr int N3_WS = N3_WC + 1;                           // odd row stride: the lanes' rows fall in different banks
constexpr int N3_WELEMS = (N3_WR * N3_WS + 15) / 16 * 16;  // one window plane, padded so the taps stay vector-aligned

// output planes (x) per CTA: as many as the registers allow without spilling at two CTAs per SM.  The forward holds
// acc[TX][RT], the adjoint acc[TX][RT] and v[TX][RT] (-Xptxas -v, sm_90a: f32 forward 4, adjoint 2; f64 1 and 1)
template <typename T, bool ADJ>
constexpr int N3_TX = sizeof(T) == 4 ? (ADJ ? 2 : 4) : 1;

// coordinates are 32-bit: in 64 bits the third axis's state does not fit the registers (every variant spilled)
struct Ns3Params {
  AxisT<int> ax[3];      // x, y, z
  int tiles_y, tiles_z;
  int n_inner;
};

template <typename T, bool ADJ>
__global__ void __launch_bounds__(NS_THREADS, 2)
ns3_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ hs, const Ns3Params p) {
  constexpr int TX = N3_TX<T, ADJ>;
  constexpr int NP = TX + N3_KCX - 1;                               // window planes of a full x chunk
  extern __shared__ __align__(64) unsigned char ns3_smem[];
  T* w = reinterpret_cast<T*>(ns3_smem);                            // [2][WR][WS] window planes (double buffer)
  T* hk = w + 2 * N3_WELEMS;                                        // [KCX][KC][KC] taps of the chunk
  double* wgx = reinterpret_cast<double*>(hk + N3_KCX * N3_KC * N3_KC);   // [NP] x weights of the planes (forward)
  double* wgy = wgx + NP;                                           // [WR] y weights of the rows (forward)
  double* wgz = wgy + N3_WR;                                        // [WC] z weights of the columns (forward)

  const auto& X = p.ax[0];
  const auto& Y = p.ax[1];
  const auto& Z = p.ax[2];
  const int ci = blockIdx.y;
  const int tyz = p.tiles_y * p.tiles_z;
  const int bx = blockIdx.x / tyz, byz = blockIdx.x % tyz;
  const int i0x = bx * TX, i0y = (byz / p.tiles_z) * N3_TY, i0z = (byz % p.tiles_z) * NS_TZ;
  const int tid = threadIdx.x, lane = tid % NS_LANES, t0 = tid / NS_LANES * NS_RT;
  // window origin (sample of plane / row / column 0) and the filters whose support can reach the tile
  const int jbx = ADJ ? i0x - X.hc : i0x + X.hc - X.nh + 1;
  const int jby = ADJ ? i0y - Y.hc : i0y + Y.hc - Y.nh + 1;
  const int jbz = ADJ ? i0z - Z.hc : i0z + Z.hc - Z.nh + 1;
  int af[3], al[3];
  {
    const int lo[3] = {ADJ ? i0x : jbx, ADJ ? i0y : jby, ADJ ? i0z : jbz};
    const int hi[3] = {ADJ ? i0x + TX : jbx + TX + X.nh - 1, ADJ ? i0y + N3_TY : jby + N3_TY + Y.nh - 1,
                             ADJ ? i0z + NS_TZ : jbz + NS_TZ + Z.nh - 1};
#pragma unroll
    for (int d = 0; d < 3; ++d) filter_span(p.ax[d], lo[d], hi[d], af[d], al[d]);
  }
  T acc[TX][NS_RT];
#pragma unroll
  for (int t = 0; t < TX; ++t)
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) acc[t][r] = T(0);

  for (int a = af[0]; a <= al[0]; ++a) {
    int qxlo, qxhi;
    if (!tap_span(X, a, i0x, jbx, TX, ADJ, qxlo, qxhi)) continue;
    int sxlo, sxhi;
    support(X, a, sxlo, sxhi);
    for (int b = af[1]; b <= al[1]; ++b) {
      int qylo, qyhi;
      if (!tap_span(Y, b, i0y, jby, N3_TY, ADJ, qylo, qyhi)) continue;
      int sylo, syhi;
      support(Y, b, sylo, syhi);
      for (int e = af[2]; e <= al[2]; ++e) {
        int qzlo, qzhi;
        if (!tap_span(Z, e, i0z, jbz, NS_TZ, ADJ, qzlo, qzhi)) continue;
        int szlo, szhi;
        support(Z, e, szlo, szhi);
        const T* hc = hs + (((size_t)a * Y.nf + b) * Z.nf + e) * (size_t)X.nh * Y.nh * Z.nh;
        T v[TX][NS_RT];
#pragma unroll
        for (int t = 0; t < TX; ++t)
#pragma unroll
          for (int r = 0; r < NS_RT; ++r) v[t][r] = T(0);
        for (int cx = qxlo; cx < qxhi; cx += N3_KCX) {
          const int nqx = min(N3_KCX, qxhi - cx);
          const int np = TX + nqx - 1;                              // window planes the chunk reads
          for (int cy = qylo; cy < qyhi; cy += N3_KC) {
            const int nqy = min(N3_KC, qyhi - cy);
            const int nwr = N3_TY + nqy - 1;                        // window rows the chunk reads
            for (int cz = qzlo; cz < qzhi; cz += N3_KC) {
              const int nqz = min(N3_KC, qzhi - cz), nqz8 = (nqz + NS_RT - 1) / NS_RT * NS_RT;
              const int nwc = NS_TZ + nqz - 1;                      // window columns with a non-zero tap
              __syncthreads();                                      // the previous chunk's readers are done
              if constexpr (!ADJ) {
                for (int m = tid; m < NP + N3_WR + N3_WC; m += NS_THREADS) {
                  if (m < NP) {
                    const int j = jbx + cx + m;
                    wgx[m] = (j >= sxlo && j < sxhi) ? axis_weight(X, a, j) : 0.0;
                  } else if (m < NP + N3_WR) {
                    const int j = jby + cy + (m - NP);
                    wgy[m - NP] = (j >= sylo && j < syhi) ? axis_weight(Y, b, j) : 0.0;
                  } else {
                    const int j = jbz + cz + (m - NP - N3_WR);
                    wgz[m - NP - N3_WR] = (j >= szlo && j < szhi) ? axis_weight(Z, e, j) : 0.0;
                  }
                }
              }
              for (int s = tid; s < nqx * N3_KC * N3_KC; s += NS_THREADS) {
                const int qx = s / (N3_KC * N3_KC), qy = s / N3_KC % N3_KC, qz = s % N3_KC;
                T tap = T(0);
                if (qy < nqy && qz < nqz) {
                  const int kx = ADJ ? cx + qx : X.nh - 1 - (cx + qx);
                  const int ky = ADJ ? cy + qy : Y.nh - 1 - (cy + qy);
                  const int kz = ADJ ? cz + qz : Z.nh - 1 - (cz + qz);
                  tap = __ldg(hc + ((size_t)kx * Y.nh + ky) * Z.nh + kz);
                }
                hk[s] = tap;
              }
              if constexpr (!ADJ) __syncthreads();                  // the weights are read by the staging below
              for (int m = 0; m < np; ++m) {
                T* wm = w + (m & 1) * N3_WELEMS;
                const int jx = jbx + cx + m;
                const bool in_x = ADJ ? (jx >= 0 && jx < X.n) : wgx[m] != 0.0;
                for (int s = tid; s < nwr * N3_WC; s += NS_THREADS) {
                  const int r = s / N3_WC, c = s - r * N3_WC;
                  const int jy = jby + cy + r, jz = jbz + cz + c;
                  T val = T(0);
                  if (in_x && c < nwc) {
                    if constexpr (ADJ) {
                      if (jy >= 0 && jy < Y.n && jz >= 0 && jz < Z.n)
                        val = __ldg(x + (((size_t)jx * Y.n + jy) * Z.n + jz) * p.n_inner + ci);
                    } else {
                      const double wy = wgy[r], wz = wgz[c];
                      if (wy != 0.0 && wz != 0.0)
                        val = T(wz * wy * wgx[m]) * __ldg(x + (((size_t)jx * Y.n + jy) * Z.n + jz) * p.n_inner + ci);
                    }
                  }
                  wm[r * N3_WS + c] = val;
                }
                __syncthreads();                                    // plane m staged; plane m - 1's readers are done
                if (!in_x) continue;                                // an all-zero plane adds nothing
                if constexpr (ADJ) correlate_plane<T, TX, N3_KC, N3_WS>(v, wm, hk, m, nqx, nqy, nqz8, lane, t0);
                else correlate_plane<T, TX, N3_KC, N3_WS>(acc, wm, hk, m, nqx, nqy, nqz8, lane, t0);
              }
            }
          }
        }
        if constexpr (ADJ) {                                        // acc += W_c v on the outputs in the support
          const int jy = i0y + lane;
          if (jy >= sylo && jy < syhi) {
            const double wy = axis_weight(Y, b, jy);
#pragma unroll
            for (int t = 0; t < TX; ++t) {
              const int jx = i0x + t;
              if (jx < sxlo || jx >= sxhi) continue;
              const double wx = axis_weight(X, a, jx);
#pragma unroll
              for (int r = 0; r < NS_RT; ++r) {
                const int jz = i0z + t0 + r;
                if (jz >= szlo && jz < szhi) acc[t][r] = fma(T(axis_weight(Z, e, jz) * wy * wx), v[t][r], acc[t][r]);
              }
            }
          }
        }
      }
    }
  }
  const int iy = i0y + lane;
  if (iy >= Y.n) return;
#pragma unroll
  for (int t = 0; t < TX; ++t) {
    const int ix = i0x + t;
    if (ix >= X.n) break;
#pragma unroll
    for (int r = 0; r < NS_RT; ++r) {
      const int iz = i0z + t0 + r;
      if (iz < Z.n) __stcs(y + (((size_t)ix * Y.n + iy) * Z.n + iz) * p.n_inner + ci, acc[t][r]);
    }
  }
}

template <typename T, bool ADJ>
int launch_ns3(const void* x, void* y, const void* hs, const Ns3Params& p, size_t nx, cudaStream_t st) {
  constexpr int TX = N3_TX<T, ADJ>;
  const long long tiles_x = (long long)((nx + TX - 1) / TX);
  if (tiles_x > 0x7fffffffLL / ((long long)p.tiles_y * p.tiles_z)) return B2_ERR_ARG;   // one 1-D grid holds every tile
  constexpr int NP = TX + N3_KCX - 1;
  const size_t smem = (size_t)(2 * N3_WELEMS + N3_KCX * N3_KC * N3_KC) * sizeof(T) +
                      (size_t)(NP + N3_WR + N3_WC) * sizeof(double);
  const int rc = b2_allow_smem<ns3_kernel<T, ADJ>>(smem);
  if (rc != B2_OK) return rc;
  ns3_kernel<T, ADJ><<<dim3((unsigned)(tiles_x * p.tiles_y * p.tiles_z), (unsigned)p.n_inner), NS_THREADS, smem, st>>>(
      static_cast<const T*>(x), static_cast<T*>(y), static_cast<const T*>(hs), p);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

}  // namespace

extern "C" int b2_nsconvolve3d(b2_ctx* ctx, const void* x, void* y, size_t nx, size_t ny, size_t nz, size_t n_inner,
                               const void* hs, int nfx, int nfy, int nfz, int nhx, int nhy, int nhz, long long ohx,
                               long long dhx, long long ohy, long long dhy, long long ohz, long long dhz, int adjoint,
                               int dtype, void* stream) {
  if (!ctx || !x || !y || !hs || x == y || (n_inner != 1 && n_inner != 2)) return B2_ERR_ARG;
  Ns3Params p;   // 32-bit axes: make_axis refuses an axis, filter size or node position of 2^29 samples or more
  if (!make_axis(nx, nfx, nhx, ohx, dhx, p.ax[0]) || !make_axis(ny, nfy, nhy, ohy, dhy, p.ax[1]) ||
      !make_axis(nz, nfz, nhz, ohz, dhz, p.ax[2]))
    return B2_ERR_ARG;
  p.n_inner = (int)n_inner;
  p.tiles_y = (int)((ny + N3_TY - 1) / N3_TY);
  p.tiles_z = (int)((nz + NS_TZ - 1) / NS_TZ);
  return b2_dispatch_real(dtype, [&](auto t) {
    using T = decltype(t);
    return adjoint ? launch_ns3<T, true>(x, y, hs, p, nx, (cudaStream_t)stream)
                   : launch_ns3<T, false>(x, y, hs, p, nx, (cudaStream_t)stream);
  });
}
