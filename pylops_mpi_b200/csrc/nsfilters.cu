// Rank-local NON-STATIONARY FILTER ESTIMATION, adjoint: the gradient of pylops.signalprocessing.
// NonStationaryFilters2D (and, with a singleton x axis, NonStationaryFilters1D) with respect to its filter bank.  The
// forward of those operators is the non-stationary convolution of a fixed real image inp by the bank (nsconvolve2d.cu
// with x = inp and hs = the model); this file holds its exact transpose,
//   g_c[kx][kz] = sum_(j in S_c) W_c[j] inp[j] d[jx + kx - hcx][jz + kz - hcz]       (terms outside the image are 0)
// for the bank g [nfx][nfz][nhx][nhz], c = (a, b), W_c[j] = T(wx_a(jx) * wz_b(jz)) and S_c the support of filter c,
// both exactly as in nsconvolve2d.cu (ns_core.cuh): the cells around the node, to the image edge for end filters.
//
// Scheme: for each filter this is a STATIONARY correlation of d with the weighted patch u_c = W_c . inp, evaluated at
// the nhx x nhz lags: the correlation of nsconvolve2d.cu with outputs and taps swapped.  A CTA owns a 32 x 64 tile of
// one filter's taps (lanes along kx, RT = 8 consecutive kz per thread in the register sliding window) and one PART of
// that filter's support.  It walks the part in 32 x 32 chunks: u_c of the chunk goes to shared memory in the place of
// the taps and d's window at origin (chunk + tap tile - hc) in the place of the image, and correlate (ns_core.cuh)
// adds one fma per term.  The support is split into a number of parts that depends on the shape alone (enough CTAs to
// fill the GPU when there are few filters with huge supports, one part when there are many); with more than one part
// each CTA writes its partial tap tile to the workspace and a second launch folds the parts.
//
// Sum order, per tap: parts in ascending (x, z) order, the first part's sum plus each later one in turn; within a part,
// chunks in ascending (x, z) order; within a chunk, terms in ascending (x, z) order, one fma each from 0.  No atomics,
// no allocation: the bits depend only on the shape and the dtype, and repeated applies give identical bits.  The sums
// differ from pylops' loop (for each point, every filter around it) only in rounding; with exactly representable
// inputs both are exact.
#include <algorithm>

#include "ns_core.cuh"

namespace {

constexpr long long NF_TARGET_CTAS = 1024;   // a part count that reaches this many CTAs fills an H100 four times over
constexpr long long NF_MIN_CHUNKS = 4;       // but a part keeps at least this many chunks of its filter's support

struct NfPlan {
  AxisT<long long> ax[2];   // x, z
  int ktx, ktz;          // tap tiles per filter
  int px, pz;            // parts per filter along x, z
  long long cpx, cpz;    // support chunks per part along x, z
  long long grid;        // CTAs of the correlation launch
  size_t work_elems;     // partial tap tiles (0: one part, written straight into the bank)
};

// the plan of a shape; false for a shape the entry points refuse
bool nf_plan(size_t nx, size_t nz, int nfx, int nfz, int nhx, int nhz, long long ohx, long long dhx, long long ohz,
             long long dhz, NfPlan& p) {
  if (!make_axis(nx, nfx, nhx, ohx, dhx, p.ax[0]) || !make_axis(nz, nfz, nhz, ohz, dhz, p.ax[1])) return false;
  if (nx > (1ULL << 40) || nz > (1ULL << 40) || nz > (1ULL << 50) / nx) return false;   // nx nz <= 2^50: no wrap
  long long mc[2] = {1, 1};                 // the most support chunks of any filter, per axis
  for (int d = 0; d < 2; ++d)
    for (int a = 0; a < p.ax[d].nf; ++a) {
      long long lo, hi;
      support(p.ax[d], a, lo, hi);
      mc[d] = std::max(mc[d], (hi - lo + N2_KC - 1) / N2_KC);
    }
  p.ktx = (nhx + N2_TX - 1) / N2_TX;
  p.ktz = (nhz + NS_TZ - 1) / NS_TZ;
  const long long base = (long long)nfx * nfz * p.ktx * p.ktz;
  long long want = std::min((NF_TARGET_CTAS + base - 1) / base, std::max(mc[0] * mc[1] / NF_MIN_CHUNKS, 1LL));
  p.cpx = (mc[0] + std::min(mc[0], want) - 1) / std::min(mc[0], want);
  p.px = (int)((mc[0] + p.cpx - 1) / p.cpx);
  want = (want + p.px - 1) / p.px;
  p.cpz = (mc[1] + std::min(mc[1], want) - 1) / std::min(mc[1], want);
  p.pz = (int)((mc[1] + p.cpz - 1) / p.cpz);
  const long long parts = (long long)p.px * p.pz;
  if (base > 0x7fffffffLL / parts) return false;            // one 1-D grid holds every CTA
  p.grid = base * parts;
  p.work_elems = parts > 1 ? (size_t)nfx * nfz * parts * nhx * nhz : 0;
  return true;
}

template <typename T>
__global__ void __launch_bounds__(NS_THREADS, 2)
nf_kernel(const T* __restrict__ d, const T* __restrict__ inp, T* __restrict__ out, const NfPlan p) {
  extern __shared__ __align__(64) unsigned char nf_smem[];
  T* w = reinterpret_cast<T*>(nf_smem);                          // [WR][WS] window of d
  T* uk = w + N2_WELEMS;                                           // [KC][KC] u_c of the chunk
  double* wgx = reinterpret_cast<double*>(uk + N2_KC * N2_KC);     // [KC] x weights of the chunk's rows
  double* wgz = wgx + N2_KC;                                       // [KC] z weights of the chunk's columns

  const auto& X = p.ax[0];
  const auto& Z = p.ax[1];
  const int parts = p.px * p.pz;
  long long idx = blockIdx.x;
  const int part = (int)(idx % parts);
  idx /= parts;
  const int tile = (int)(idx % (p.ktx * p.ktz));
  const long long c = idx / (p.ktx * p.ktz);
  const int a = (int)(c / Z.nf), b = (int)(c % Z.nf);
  const int k0x = tile / p.ktz * N2_TX, k0z = tile % p.ktz * NS_TZ;
  const int tid = threadIdx.x, lane = tid % NS_LANES, t0 = tid / NS_LANES * NS_RT;

  long long sxlo, sxhi, szlo, szhi;
  support(X, a, sxlo, sxhi);
  support(Z, b, szlo, szhi);
  const long long jxlo = sxlo + part / p.pz * p.cpx * N2_KC, jxhi = min(sxhi, jxlo + p.cpx * N2_KC);
  const long long jzlo = szlo + part % p.pz * p.cpz * N2_KC, jzhi = min(szhi, jzlo + p.cpz * N2_KC);

  T acc[NS_RT];
#pragma unroll
  for (int r = 0; r < NS_RT; ++r) acc[r] = T(0);

  for (long long jx0 = jxlo; jx0 < jxhi; jx0 += N2_KC) {
    const int nqx = (int)min((long long)N2_KC, jxhi - jx0);
    const int nwr = N2_TX + nqx - 1;                               // window rows the chunk reads
    const long long ox = jx0 + k0x - X.hc;                         // sample of window row 0
    if (ox >= X.n || ox + nwr <= 0) continue;                      // every term of the chunk is 0
    for (long long jz0 = jzlo; jz0 < jzhi; jz0 += N2_KC) {
      const int nqz = (int)min((long long)N2_KC, jzhi - jz0), nqz8 = (nqz + NS_RT - 1) / NS_RT * NS_RT;
      const int nwc = NS_TZ + nqz - 1;                             // window columns a non-zero u meets
      const long long oz = jz0 + k0z - Z.hc;
      if (oz >= Z.n || oz + nwc <= 0) continue;
      __syncthreads();                                             // the previous chunk's readers are done
      if (tid < 2 * N2_KC) {
        const int m = tid % N2_KC;
        if (tid < N2_KC) wgx[m] = m < nqx ? axis_weight(X, a, jx0 + m) : 0.0;
        else wgz[m] = m < nqz ? axis_weight(Z, b, jz0 + m) : 0.0;
      }
      for (int e = tid; e < nwr * N2_WC; e += NS_THREADS) {
        const int r = e / N2_WC, col = e - r * N2_WC;
        const long long jx = ox + r, jz = oz + col;
        T val = T(0);
        if (col < nwc && jx >= 0 && jx < X.n && jz >= 0 && jz < Z.n) val = __ldg(d + (size_t)jx * Z.n + jz);
        w[r * N2_WS + col] = val;
      }
      __syncthreads();                                             // the weights are in
      for (int e = tid; e < nqx * N2_KC; e += NS_THREADS) {
        const int qx = e / N2_KC, qz = e - qx * N2_KC;
        T val = T(0);
        if (qz < nqz) val = T(wgz[qz] * wgx[qx]) * __ldg(inp + (size_t)(jx0 + qx) * Z.n + (jz0 + qz));
        uk[e] = val;
      }
      __syncthreads();
      correlate<T>(acc, w, uk, nqx, nqz8, lane, t0);
    }
  }
  const int kx = k0x + lane;
  if (kx >= X.nh) return;
  T* dst = out + ((size_t)c * parts + part) * X.nh * Z.nh + (size_t)kx * Z.nh;
#pragma unroll
  for (int r = 0; r < NS_RT; ++r) {
    const int kz = k0z + t0 + r;
    if (kz < Z.nh) dst[kz] = acc[r];
  }
}

// hs[c][k] = sum over the parts q of work[c][q][k], in ascending q
template <typename T>
__global__ void __launch_bounds__(256)
nf_fold_kernel(const T* __restrict__ work, T* __restrict__ hs, size_t n, size_t nh, int parts) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const T* src = work + (i / nh * parts) * nh + i % nh;
    T s = src[0];
    for (int q = 1; q < parts; ++q) s += src[(size_t)q * nh];
    hs[i] = s;
  }
}

template <typename T>
int launch_nf(const void* d, const void* inp, void* hs, void* work, const NfPlan& p, cudaStream_t st) {
  const size_t smem = (size_t)(N2_WELEMS + N2_KC * N2_KC) * sizeof(T) + (size_t)(2 * N2_KC) * sizeof(double);
  const int rc = b2_allow_smem<nf_kernel<T>>(smem);
  if (rc != B2_OK) return rc;
  T* dst = static_cast<T*>(p.work_elems ? work : hs);
  nf_kernel<T><<<(unsigned)p.grid, NS_THREADS, smem, st>>>(static_cast<const T*>(d), static_cast<const T*>(inp), dst,
                                                           p);
  B2_LAUNCH_CHECK();
  if (p.work_elems) {
    const size_t n = (size_t)p.ax[0].nf * p.ax[1].nf * p.ax[0].nh * p.ax[1].nh;
    const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, 4096);
    nf_fold_kernel<T><<<blocks, 256, 0, st>>>(dst, static_cast<T*>(hs), n, (size_t)p.ax[0].nh * p.ax[1].nh,
                                              p.px * p.pz);
    B2_LAUNCH_CHECK();
  }
  return B2_OK;
}

bool overlap(const void* a, size_t na, const void* b, size_t nb) {
  const char *pa = static_cast<const char*>(a), *pb = static_cast<const char*>(b);
  return pa < pb + nb && pb < pa + na;
}

size_t real_size(int dtype) { return dtype == B2_F32 ? 4 : dtype == B2_F64 ? 8 : 0; }

}  // namespace

extern "C" int b2_nsfilters2d_work_bytes(size_t nx, size_t nz, int nfx, int nfz, int nhx, int nhz, long long ohx,
                                         long long dhx, long long ohz, long long dhz, int dtype, size_t* bytes) {
  if (!bytes) return B2_ERR_ARG;
  if (!real_size(dtype)) return B2_ERR_DTYPE;
  NfPlan p;
  if (!nf_plan(nx, nz, nfx, nfz, nhx, nhz, ohx, dhx, ohz, dhz, p)) return B2_ERR_ARG;
  *bytes = p.work_elems * real_size(dtype);
  return B2_OK;
}

extern "C" int b2_nsfilters2d_adjoint(b2_ctx* ctx, const void* d, const void* inp, void* hs_out, size_t nx, size_t nz,
                                      int nfx, int nfz, int nhx, int nhz, long long ohx, long long dhx, long long ohz,
                                      long long dhz, void* work, size_t work_bytes, int dtype, void* stream) {
  if (!ctx || !d || !inp || !hs_out) return B2_ERR_ARG;
  const size_t es = real_size(dtype);
  if (!es) return B2_ERR_DTYPE;
  NfPlan p;
  if (!nf_plan(nx, nz, nfx, nfz, nhx, nhz, ohx, dhx, ohz, dhz, p)) return B2_ERR_ARG;
  const size_t nimg = nx * nz * es, nbank = (size_t)nfx * nfz * nhx * nhz * es, nwork = p.work_elems * es;
  if (overlap(hs_out, nbank, d, nimg) || overlap(hs_out, nbank, inp, nimg)) return B2_ERR_ARG;
  if (nwork) {
    if (!work || work_bytes < nwork) return B2_ERR_ARG;
    if (overlap(work, nwork, d, nimg) || overlap(work, nwork, inp, nimg) || overlap(work, nwork, hs_out, nbank))
      return B2_ERR_ARG;
  }
  return b2_dispatch_real(dtype, [&](auto t) {
    return launch_nf<decltype(t)>(d, inp, hs_out, work, p, (cudaStream_t)stream);
  });
}
