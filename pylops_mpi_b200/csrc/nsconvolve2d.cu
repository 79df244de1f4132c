// Rank-local NON-STATIONARY 2-D convolution of a C-ordered [nx][nz][n_inner] image: the role of
// pylops.signalprocessing.NonStationaryConvolve2D inside MPIBlockDiag (n_inner = 2: complex data as (re, im) pairs).
//
// Filter bank hs [nfx][nfz][nhx][nhz] at the image points (ohx + a dhx, ohz + b dhz), centre (hcx, hcz) = (nhx / 2,
// nhz / 2).  Point j = (jx, jz) uses h_j = sum_(a,b) W_ab[j] hs[a][b], with separable bilinear weights
//   W_ab[j] = T(wx_a(jx) * wz_b(jz))   (the float64 product rounded to the data type T)
// and per axis  v = (j - oh) / dh (float64), l = floor(v), w = v - l:  weight 1 on filter 0 (l < 0) or on filter nf - 1
// (l >= nf - 1), else 1 - w on l and w on l + 1.
//   forward  y[i] = sum_j h_j[hc + i - j] x[j]       (a scatter: point j spreads its own filter)
//   adjoint  x[j] = sum_i h_j[hc + i - j] y[i]       (the exact transpose)
// Points outside the image are zero.
//
// Scheme: the bilinear decomposition.  Since h_j is linear in the bank,
//   forward  y = sum_c h_c * (W_c . x)               adjoint  x = sum_c W_c . (h_c (x) y)
// (c = (a, b) over the bank, * convolution, (x) correlation, . the point-wise product).  W_c is non-zero only on the
// support S_c of filter c (the cells around its node), so a CTA of 32 x 64 outputs runs, for each filter whose support
// reaches it, one STATIONARY correlation restricted to the taps that can meet the support: every tap it reads is a
// broadcast and every term is one fma, against about eight operations per term for a tap interpolated per (point,
// tap) pair.  Lanes of a warp run along x (one output row each) and a thread's RT = 8 consecutive z outputs slide a
// register window along z, as in nsconvolve.cu; the window row stride is odd, so the lanes' rows never share a bank.
// Taps are processed in chunks of KC x KC: any filter size fits the fixed shared memory.
//   forward  the window holds u_c = W_c . x (zero off S_c) and the taps are reversed: acc[t] += h_c[K-1-q] u_c[t + q]
//   adjoint  the window holds y, v[t] += h_c[q] y[t + q] over the whole filter, then acc[t] = fma(W_c[t], v[t], acc[t])
// Sum order: filters in ascending (a, b); within a filter, tap chunks in ascending (x, z) order and the taps of a chunk
// in ascending (x, z) order (forward: of the reversed filter), one fma per term.  No atomics, no allocation: repeated
// applies give identical bits.  The sums differ from pylops' (interpolate h_j, then convolve) only in rounding; with
// exactly representable inputs both are exact.
#include "ns_core.cuh"

namespace {

struct Ns2Params {
  AxisT<long long> ax[2];   // x, z
  long long tiles_z;
  long long n_inner;
};

template <typename T, bool ADJ>
__global__ void __launch_bounds__(NS_THREADS, 2)
ns2_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ hs, const Ns2Params p) {
  extern __shared__ __align__(64) unsigned char ns2_smem[];
  T* w = reinterpret_cast<T*>(ns2_smem);                          // [WR][WS] window
  T* hk = w + N2_WELEMS;                                           // [KC][KC] taps of the chunk
  double* wgx = reinterpret_cast<double*>(hk + N2_KC * N2_KC);     // [WR] x weights of the window rows (forward)
  double* wgz = wgx + N2_WR;                                       // [WC] z weights of the window columns (forward)

  const auto& X = p.ax[0];
  const auto& Z = p.ax[1];
  const long long ci = blockIdx.y;
  const long long i0x = (long long)(blockIdx.x / p.tiles_z) * N2_TX, i0z = (long long)(blockIdx.x % p.tiles_z) * NS_TZ;
  const int tid = threadIdx.x, lane = tid % NS_LANES, t0 = tid / NS_LANES * NS_RT;
  // window origin (sample of row / column 0) and the filters whose support can reach the tile
  const long long jbx = ADJ ? i0x - X.hc : i0x + X.hc - X.nh + 1;
  const long long jbz = ADJ ? i0z - Z.hc : i0z + Z.hc - Z.nh + 1;
  int af[2], al[2];
  {
    const long long lo[2] = {ADJ ? i0x : jbx, ADJ ? i0z : jbz};
    const long long hi[2] = {ADJ ? i0x + N2_TX : jbx + N2_TX + X.nh - 1, ADJ ? i0z + NS_TZ : jbz + NS_TZ + Z.nh - 1};
#pragma unroll
    for (int d = 0; d < 2; ++d) filter_span(p.ax[d], lo[d], hi[d], af[d], al[d]);
  }
  T acc[NS_RT];
#pragma unroll
  for (int r = 0; r < NS_RT; ++r) acc[r] = T(0);

  for (int a = af[0]; a <= al[0]; ++a) {
    int qxlo, qxhi;
    if (!tap_span(X, a, i0x, jbx, N2_TX, ADJ, qxlo, qxhi)) continue;
    long long sxlo, sxhi;
    support(X, a, sxlo, sxhi);
    for (int b = af[1]; b <= al[1]; ++b) {
      int qzlo, qzhi;
      if (!tap_span(Z, b, i0z, jbz, NS_TZ, ADJ, qzlo, qzhi)) continue;
      long long szlo, szhi;
      support(Z, b, szlo, szhi);
      const T* hc = hs + ((size_t)a * Z.nf + b) * (size_t)X.nh * Z.nh;
      T v[NS_RT];
#pragma unroll
      for (int r = 0; r < NS_RT; ++r) v[r] = T(0);
      for (int cx = qxlo; cx < qxhi; cx += N2_KC) {
        const int nqx = min(N2_KC, qxhi - cx);
        const int nwr = N2_TX + nqx - 1;                            // window rows the chunk reads
        for (int cz = qzlo; cz < qzhi; cz += N2_KC) {
          const int nqz = min(N2_KC, qzhi - cz), nqz8 = (nqz + NS_RT - 1) / NS_RT * NS_RT;
          const int nwc = NS_TZ + nqz - 1;                          // window columns with a non-zero tap
          __syncthreads();                                          // the previous chunk's readers are done
          if constexpr (!ADJ) {
            for (int m = tid; m < N2_WR + N2_WC; m += NS_THREADS) {
              if (m < N2_WR) {
                const long long j = jbx + cx + m;
                wgx[m] = (j >= sxlo && j < sxhi) ? axis_weight(X, a, j) : 0.0;
              } else {
                const long long j = jbz + cz + (m - N2_WR);
                wgz[m - N2_WR] = (j >= szlo && j < szhi) ? axis_weight(Z, b, j) : 0.0;
              }
            }
            __syncthreads();
          }
          for (int e = tid; e < nwr * N2_WC; e += NS_THREADS) {
            const int r = e / N2_WC, c = e - r * N2_WC;
            const long long jx = jbx + cx + r, jz = jbz + cz + c;
            T val = T(0);
            if (c < nwc) {
              if constexpr (ADJ) {
                if (jx >= 0 && jx < X.n && jz >= 0 && jz < Z.n)
                  val = __ldg(x + ((size_t)jx * Z.n + jz) * p.n_inner + ci);
              } else {
                const double wx = wgx[r], wz = wgz[c];
                if (wx != 0.0 && wz != 0.0)
                  val = T(wz * wx) * __ldg(x + ((size_t)jx * Z.n + jz) * p.n_inner + ci);
              }
            }
            w[r * N2_WS + c] = val;
          }
          for (int e = tid; e < nqx * N2_KC; e += NS_THREADS) {
            const int qx = e / N2_KC, qz = e - qx * N2_KC;
            T tap = T(0);
            if (qz < nqz) {
              const int kx = ADJ ? cx + qx : X.nh - 1 - (cx + qx), kz = ADJ ? cz + qz : Z.nh - 1 - (cz + qz);
              tap = __ldg(hc + (size_t)kx * Z.nh + kz);
            }
            hk[e] = tap;
          }
          __syncthreads();
          if constexpr (ADJ) correlate<T>(v, w, hk, nqx, nqz8, lane, t0);
          else correlate<T>(acc, w, hk, nqx, nqz8, lane, t0);
        }
      }
      if constexpr (ADJ) {                                          // acc += W_c v on the outputs in the support
        const long long jx = i0x + lane;
        if (jx >= sxlo && jx < sxhi) {
          const double wx = axis_weight(X, a, jx);
#pragma unroll
          for (int r = 0; r < NS_RT; ++r) {
            const long long jz = i0z + t0 + r;
            if (jz >= szlo && jz < szhi) acc[r] = fma(T(axis_weight(Z, b, jz) * wx), v[r], acc[r]);
          }
        }
      }
    }
  }
  const long long ix = i0x + lane;
  if (ix >= X.n) return;
#pragma unroll
  for (int r = 0; r < NS_RT; ++r) {
    const long long iz = i0z + t0 + r;
    if (iz < Z.n) __stcs(y + ((size_t)ix * Z.n + iz) * p.n_inner + ci, acc[r]);
  }
}

template <typename T, bool ADJ>
int launch_ns2(const void* x, void* y, const void* hs, const Ns2Params& p, long long tiles_x, cudaStream_t st) {
  const size_t smem = (size_t)(N2_WELEMS + N2_KC * N2_KC) * sizeof(T) + (size_t)(N2_WR + N2_WC) * sizeof(double);
  const int rc = b2_allow_smem<ns2_kernel<T, ADJ>>(smem);
  if (rc != B2_OK) return rc;
  ns2_kernel<T, ADJ><<<dim3((unsigned)(tiles_x * p.tiles_z), (unsigned)p.n_inner), NS_THREADS, smem, st>>>(
      static_cast<const T*>(x), static_cast<T*>(y), static_cast<const T*>(hs), p);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

}  // namespace

extern "C" int b2_nsconvolve2d(b2_ctx* ctx, const void* x, void* y, size_t nx, size_t nz, size_t n_inner,
                               const void* hs, int nfx, int nfz, int nhx, int nhz, long long ohx, long long dhx,
                               long long ohz, long long dhz, int adjoint, int dtype, void* stream) {
  if (!ctx || !x || !y || !hs || x == y || (n_inner != 1 && n_inner != 2)) return B2_ERR_ARG;
  Ns2Params p;
  if (!make_axis(nx, nfx, nhx, ohx, dhx, p.ax[0]) || !make_axis(nz, nfz, nhz, ohz, dhz, p.ax[1])) return B2_ERR_ARG;
  p.n_inner = (long long)n_inner;
  p.tiles_z = (long long)((nz + NS_TZ - 1) / NS_TZ);
  const long long tiles_x = (long long)((nx + N2_TX - 1) / N2_TX);
  if (tiles_x > 0x7fffffffLL / p.tiles_z) return B2_ERR_ARG;      // one 1-D grid holds every tile
  return b2_dispatch_real(dtype, [&](auto t) {
    using T = decltype(t);
    return adjoint ? launch_ns2<T, true>(x, y, hs, p, tiles_x, (cudaStream_t)stream)
                   : launch_ns2<T, false>(x, y, hs, p, tiles_x, (cudaStream_t)stream);
  });
}
