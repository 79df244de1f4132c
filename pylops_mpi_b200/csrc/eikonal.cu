// Eikonal traveltime tables (b2_eikonal_tables): the first-arrival traveltime from each of n grid nodes through a
// velocity model on the image grid, for pylops.waveeqprocessing.Kirchhoff(mode="eikonal") with the tables in
// b2_kirchhoff's layout table[p][ii] (ii = (iy * nx + ix) * nz + iz; 2-D is ny = 1).
//
// The discrete problem, exactly.  T_0 = 0 at the point's node, +inf elsewhere.  One Jacobi step computes every node's
// new value from the previous iterate only:
//   s = 1 / vel[node]                                  (correctly rounded divide, once per node)
//   a_y, a_x, a_z = the smaller of the two neighbours' old values along each axis (a neighbour off the grid is +inf)
//   (a_k, h_k, w_k) with w_k = 1 / (h_k * h_k) for h = (dy, dx, dz), stably sorted by a_k (ties keep y, x, z order):
//   a1 <= a2 <= a3
//   t = a1 + h1 * s
//   if t > a2:                                         two axes, larger root of sum_k w_k (t - a_k)^2 = s^2
//     d2 = a2 - a1, p2 = w2 * d2, q2 = p2 * d2
//     A = w1 + w2, B = p2, C = q2 - s * s
//     t = a1 + (B + sqrt(max(B * B - A * C, 0))) / A
//     if t > a3:                                       three axes
//       d3 = a3 - a1, p3 = w3 * d3, q3 = p3 * d3
//       A = (w1 + w2) + w3, B = p2 + p3, C = (q2 + q3) - s * s
//       t = a1 + (B + sqrt(max(B * B - A * C, 0))) / A
//   new = min(old, t)
// Every operation is one IEEE float64 operation, rounded to nearest (explicit intrinsics: no fma contraction), so
// the iterate equals the vectorised NumPy restatement (tests/golden/refshim/pylops/waveeqprocessing/eikonal.py) bit
// for bit.  The values only decrease and the update is monotone, so the iteration stops at the fixed point; the
// result is the iterate after max_iter steps, which is the fixed point whenever that was reached by then.
//
// Temporal blocking.  A CTA owns one tile of one field: it loads the tile plus a halo of K cells (off-grid cells are
// +inf) into shared memory and runs k <= K Jacobi steps there, ping-ponging two shared buffers; step j recomputes the
// cells at least j cells from the box's faces, so after k steps the tile's values equal k global Jacobi steps
// exactly.  It writes the tile to the other global buffer (global ping-pong, so no CTA reads what another writes in
// the same pass).
//
// Active tiles.  A tile is recomputed only if it or one of its 3^d neighbours changed in the previous pass: the box
// (tile + halo, K <= the tile edge) then holds the same values as at the start of that pass, and since values only
// decrease, a tile that k' steps did not change stays unchanged for any k <= k' steps.  Passes therefore run k = K
// steps and only the last (max_iter not a multiple of K) fewer.  The output buffer of a skipped tile already holds
// its values (they did not change in the previous pass, whose input that buffer was).
//
// All fields (points) run in one grid, blockIdx = (tile, field).  One device word records the last step that changed
// a value; the host reads it every EK_CHECK passes (a pass after the fixed point changes nothing and costs one flag
// check per CTA).  When max_iter steps end without a pass that changed nothing, one more step into the spare buffer
// decides between B2_OK and B2_ERR_CONVERGE.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int EK_THREADS = 256;
constexpr int EK_CHECK = 4;          // passes between host reads of the progress word
constexpr int EK_INIT_THREADS = 256;

// interior (TY, TX, TZ) and halo K (= steps per pass) of one tile; 2-D (ny = 1) has no y halo
template <int D>
struct Tile;
template <>
struct Tile<2> {
  static constexpr int TY = 1, TX = 32, TZ = 32, K = 8, HY = 0;
};
template <>
struct Tile<3> {
  static constexpr int TY = 8, TX = 8, TZ = 8, K = 4, HY = 4;
};
template <int D>
struct Box {
  using T = Tile<D>;
  static constexpr int BY = T::TY + 2 * T::HY, BX = T::TX + 2 * T::K, BZ = T::TZ + 2 * T::K;
  static constexpr int N = BY * BX * BZ;
  static constexpr size_t SMEM = 2 * N * sizeof(double);
};

struct Geom {
  int ny, nx, nz, nty, ntx, ntz;                         // grid and tile counts per axis (each < 2^31)
  long long ni, ntiles;
  double h[3], w[3];   // spacings (y, x, z) and 1 / h^2
};

// progress words in the work buffer
enum { CTR_LAST = 0, CTR_ACTIVE = 1, CTR_BADVEL = 2, CTR_N = 4 };

__device__ __forceinline__ double dmin(double a, double b) { return b < a ? b : a; }

__device__ __forceinline__ double root(double A, double B, double C, double a1) {
  double disc = __dsub_rn(__dmul_rn(B, B), __dmul_rn(A, C));
  disc = disc > 0.0 ? disc : 0.0;
  return __dadd_rn(a1, __ddiv_rn(__dadd_rn(B, __dsqrt_rn(disc)), A));
}

// the Godunov update of the header comment
__device__ __forceinline__ double godunov(double a1, double a2, double a3, const Geom& g, double s) {
  double h1 = g.h[0], h2 = g.h[1], h3 = g.h[2], w1 = g.w[0], w2 = g.w[1], w3 = g.w[2];
#define EK_SWAP(i, j)                                                        \
  if (a##i > a##j) {                                                         \
    double t_ = a##i; a##i = a##j; a##j = t_;                                \
    t_ = h##i; h##i = h##j; h##j = t_;                                       \
    t_ = w##i; w##i = w##j; w##j = t_;                                       \
  }
  EK_SWAP(1, 2)
  EK_SWAP(2, 3)
  EK_SWAP(1, 2)
#undef EK_SWAP
  double t = __dadd_rn(a1, __dmul_rn(h1, s));
  if (t > a2) {
    const double sq = __dmul_rn(s, s);
    const double d2 = __dsub_rn(a2, a1), p2 = __dmul_rn(w2, d2), q2 = __dmul_rn(p2, d2);
    const double A2 = __dadd_rn(w1, w2);
    t = root(A2, p2, __dsub_rn(q2, sq), a1);
    if (t > a3) {
      const double d3 = __dsub_rn(a3, a1), p3 = __dmul_rn(w3, d3), q3 = __dmul_rn(p3, d3);
      t = root(__dadd_rn(A2, w3), __dadd_rn(p2, p3), __dsub_rn(__dadd_rn(q2, q3), sq), a1);
    }
  }
  return t;
}

// s = 1 / vel; flags a velocity that is not finite and positive
__global__ void eikonal_slowness_kernel(const double* __restrict__ vel, double* __restrict__ slow, long long ni,
                                        unsigned long long* __restrict__ ctr) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < ni; i += (long long)gridDim.x * blockDim.x) {
    const double v = vel[i];
    if (!(v > 0.0) || !isfinite(v)) ctr[CTR_BADVEL] = 1ULL;
    slow[i] = __ddiv_rn(1.0, v);
  }
}

// T_0 into both global buffers; previous-pass flags: only each field's source tile "changed"
template <int D>
__global__ void eikonal_init_kernel(double* __restrict__ t0, double* __restrict__ t1, const long long* __restrict__ idx,
                                    long long n, Geom g, unsigned char* __restrict__ prev,
                                    unsigned char* __restrict__ cur) {
  using TL = Tile<D>;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long first = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long e = first; e < n * g.ni; e += stride) {
    const long long f = e / g.ni, ii = e - f * g.ni;
    const long long* p = idx + 3 * f;
    const double v = ii == (p[0] * g.nx + p[1]) * g.nz + p[2] ? 0.0 : INFINITY;
    t0[e] = v;
    t1[e] = v;
  }
  for (long long e = first; e < n * g.ntiles; e += stride) {
    const long long f = e / g.ntiles, tile = e - f * g.ntiles;
    const long long* p = idx + 3 * f;
    const long long src = ((p[0] / TL::TY) * g.ntx + p[1] / TL::TX) * g.ntz + p[2] / TL::TZ;
    prev[e] = tile == src;
    cur[e] = 0;
  }
}

// one pass: k Jacobi steps of every active (tile, field), src -> dst
template <int D>
__global__ void __launch_bounds__(EK_THREADS)
eikonal_pass_kernel(const double* __restrict__ src, double* __restrict__ dst, const double* __restrict__ slow,
                    const unsigned char* __restrict__ prev, unsigned char* __restrict__ cur,
                    unsigned long long* __restrict__ ctr, Geom g, long long n, int k, long long step0) {
  using TL = Tile<D>;
  using BB = Box<D>;
  constexpr int BY = BB::BY, BX = BB::BX, BZ = BB::BZ, NB = BB::N, NT = TL::TY * TL::TX * TL::TZ;
  constexpr int NNB = D == 3 ? 27 : 9;
  extern __shared__ double ek_smem[];
  double* const u0 = ek_smem;
  double* const u1 = ek_smem + NB;
  const int tile = blockIdx.x;
  const int tz = tile % g.ntz, tx = (tile / g.ntz) % g.ntx, ty = tile / (g.ntz * g.ntx);
  const int y0 = ty * TL::TY - TL::HY, x0 = tx * TL::TX - TL::K, z0 = tz * TL::TZ - TL::K;   // box origin

  for (long long f = blockIdx.y; f < n; f += gridDim.y) {
    const unsigned char* pf = prev + f * g.ntiles;
    int act = 0;
    if (threadIdx.x < NNB) {
      const int oy = D == 3 ? (int)threadIdx.x / 9 - 1 : 0, r = (int)threadIdx.x % 9;
      const int y = ty + oy, x = tx + r / 3 - 1, z = tz + r % 3 - 1;
      if (y >= 0 && y < g.nty && x >= 0 && x < g.ntx && z >= 0 && z < g.ntz)
        act = pf[((long long)y * g.ntx + x) * g.ntz + z];
    }
    if (!__syncthreads_or(act)) {
      if (threadIdx.x == 0) cur[f * g.ntiles + tile] = 0;
      continue;
    }
    const double* sf = src + f * g.ni;
    for (int l = threadIdx.x; l < NB; l += EK_THREADS) {
      const int by = l / (BX * BZ), bx = (l / BZ) % BX, bz = l % BZ;
      const int gy = y0 + by, gx = x0 + bx, gz = z0 + bz;
      double v = INFINITY;
      if (gy >= 0 && gy < g.ny && gx >= 0 && gx < g.nx && gz >= 0 && gz < g.nz) v = sf[((long long)gy * g.nx + gx) * g.nz + gz];
      u0[l] = v;
      u1[l] = v;
    }
    __syncthreads();
    int last = 0;                                     // last step that changed a value of the tile
    for (int j = 1; j <= k; ++j) {
      const double* o = (j & 1) ? u0 : u1;
      double* w = (j & 1) ? u1 : u0;
      int chg = 0;
      for (int l = threadIdx.x; l < NB; l += EK_THREADS) {
        const int by = l / (BX * BZ), bx = (l / BZ) % BX, bz = l % BZ;
        if (bx < j || bx >= BX - j || bz < j || bz >= BZ - j) continue;
        if (D == 3 && (by < j || by >= BY - j)) continue;
        const int gy = y0 + by, gx = x0 + bx, gz = z0 + bz;
        if (gy < 0 || gy >= g.ny || gx < 0 || gx >= g.nx || gz < 0 || gz >= g.nz) continue;
        const double old = o[l];
        const double ay = D == 3 ? dmin(o[l - BX * BZ], o[l + BX * BZ]) : INFINITY;
        const double ax = dmin(o[l - BZ], o[l + BZ]), az = dmin(o[l - 1], o[l + 1]);
        const double t = godunov(ay, ax, az, g, __ldg(slow + ((long long)gy * g.nx + gx) * g.nz + gz));
        const double nv = dmin(old, t);
        w[l] = nv;
        if (nv != old && by >= TL::HY && by < TL::HY + TL::TY && bx >= TL::K && bx < TL::K + TL::TX &&
            bz >= TL::K && bz < TL::K + TL::TZ)
          chg = 1;
      }
      if (__syncthreads_or(chg)) last = j;
    }
    const double* fin = (k & 1) ? u1 : u0;
    double* df = dst + f * g.ni;
    for (int l = threadIdx.x; l < NT; l += EK_THREADS) {
      const int iy = l / (TL::TX * TL::TZ), ix = (l / TL::TZ) % TL::TX, iz = l % TL::TZ;
      const int gy = y0 + TL::HY + iy, gx = x0 + TL::K + ix, gz = z0 + TL::K + iz;
      if (gy < g.ny && gx < g.nx && gz < g.nz)
        df[((long long)gy * g.nx + gx) * g.nz + gz] = fin[((TL::HY + iy) * BX + TL::K + ix) * BZ + TL::K + iz];
    }
    if (threadIdx.x == 0) {
      cur[f * g.ntiles + tile] = last > 0;
      if (last > 0) atomicMax(ctr + CTR_LAST, (unsigned long long)(step0 + last));
      atomicAdd(ctr + CTR_ACTIVE, 1ULL);
    }
    __syncthreads();                                  // shared buffers are reused by the next field
  }
}

Geom make_geom(size_t ny, size_t nx, size_t nz, double dy, double dx, double dz) {
  Geom g;
  const bool three = ny > 1;
  const int ty = three ? Tile<3>::TY : Tile<2>::TY, tx = three ? Tile<3>::TX : Tile<2>::TX,
            tz = three ? Tile<3>::TZ : Tile<2>::TZ;
  g.ny = (int)ny;
  g.nx = (int)nx;
  g.nz = (int)nz;
  g.ni = (long long)ny * (long long)nx * (long long)nz;
  g.nty = (g.ny + ty - 1) / ty;
  g.ntx = (g.nx + tx - 1) / tx;
  g.ntz = (g.nz + tz - 1) / tz;
  g.ntiles = (long long)g.nty * g.ntx * g.ntz;
  g.h[0] = dy;
  g.h[1] = dx;
  g.h[2] = dz;
  for (int a = 0; a < 3; ++a) g.w[a] = 1.0 / (g.h[a] * g.h[a]);   // host IEEE float64, as NumPy's 1 / (h * h)
  return g;
}

// work buffer layout: [n*ni doubles: second iterate][ni doubles: slowness][3n long long: nodes][CTR_N words]
//                     [n*ntiles bytes: flags A][n*ntiles bytes: flags B]
size_t work_bytes(const Geom& g, size_t n) {
  return ((size_t)g.ni * n + (size_t)g.ni + 3 * n + CTR_N) * 8 + 2 * n * (size_t)g.ntiles;
}

bool sizes_ok(size_t ny, size_t nx, size_t nz, size_t n) {
  if (ny == 0 || nx == 0 || nz == 0 || n == 0) return false;
  const size_t lim = (size_t)1 << 40, axis = 0x7fffffffULL;
  if (ny > axis || nx > axis || nz > axis || n > axis) return false;
  return nx < lim / nz && ny < lim / (nx * nz) && n < lim / (ny * nx * nz);
}

template <int D>
int solve(const Geom& g, const double* vel, const long long* idx_host, size_t n, size_t max_iter, double* table,
          unsigned char* work, long long* info_host, cudaStream_t st) {
  double* spare = reinterpret_cast<double*>(work);
  double* slow = spare + (size_t)g.ni * n;
  long long* idx = reinterpret_cast<long long*>(slow + g.ni);
  unsigned long long* ctr = reinterpret_cast<unsigned long long*>(idx + 3 * n);
  unsigned char* flags[2] = {reinterpret_cast<unsigned char*>(ctr + CTR_N), nullptr};
  flags[1] = flags[0] + n * (size_t)g.ntiles;
  unsigned long long h_ctr[CTR_N];

  B2_CUDA(cudaMemsetAsync(ctr, 0, CTR_N * sizeof(unsigned long long), st));
  B2_CUDA(cudaMemcpyAsync(idx, idx_host, 3 * n * sizeof(long long), cudaMemcpyHostToDevice, st));
  const long long sb = (g.ni + EK_INIT_THREADS - 1) / EK_INIT_THREADS;
  eikonal_slowness_kernel<<<(unsigned)(sb < 4096 ? sb : 4096), EK_INIT_THREADS, 0, st>>>(vel, slow, g.ni, ctr);
  B2_LAUNCH_CHECK();
  B2_CUDA(cudaMemcpyAsync(h_ctr, ctr, sizeof h_ctr, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (h_ctr[CTR_BADVEL]) return B2_ERR_ARG;                     // table untouched

  double* buf[2] = {table, spare};
  eikonal_init_kernel<D><<<4096, EK_INIT_THREADS, 0, st>>>(table, spare, idx, (long long)n, g, flags[0], flags[1]);
  B2_LAUNCH_CHECK();
  const size_t smem = Box<D>::SMEM;
  B2_CUDA(cudaFuncSetAttribute(eikonal_pass_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (g.ntiles > 0x7fffffffLL) return B2_ERR_ARG;
  const dim3 grid((unsigned)g.ntiles, (unsigned)(n < 65535 ? n : 65535));
  size_t done = 0, passes = 0;
  bool converged = false;
  auto pass = [&](int k) -> int {
    eikonal_pass_kernel<D><<<grid, EK_THREADS, smem, st>>>(buf[passes & 1], buf[(passes + 1) & 1], slow,
                                                          flags[passes & 1], flags[(passes + 1) & 1], ctr, g,
                                                          (long long)n, k, (long long)done);
    B2_LAUNCH_CHECK();
    return B2_OK;
  };
  while (done < max_iter) {
    const size_t left = max_iter - done;
    const int k = left < (size_t)Tile<D>::K ? (int)left : Tile<D>::K;
    const int rc = pass(k);
    if (rc != B2_OK) return rc;
    done += k;
    ++passes;
    if (passes % EK_CHECK == 0 || done == max_iter) {
      B2_CUDA(cudaMemcpyAsync(h_ctr, ctr, sizeof h_ctr, cudaMemcpyDeviceToHost, st));
      B2_CUDA(cudaStreamSynchronize(st));
      if (h_ctr[CTR_LAST] < done) {                             // a step changed nothing: the fixed point
        converged = true;
        break;
      }
    }
  }
  double* result = buf[passes & 1];
  const size_t run = passes;
  if (!converged) {                                             // is the max_iter-th iterate the fixed point?
    int rc = pass(1);
    if (rc != B2_OK) return rc;
    B2_CUDA(cudaMemcpyAsync(h_ctr, ctr, sizeof h_ctr, cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    converged = h_ctr[CTR_LAST] <= max_iter;
  }
  if (result != table)
    B2_CUDA(cudaMemcpyAsync(table, result, (size_t)g.ni * n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (info_host) {
    B2_CUDA(cudaStreamSynchronize(st));
    info_host[0] = (long long)(h_ctr[CTR_LAST] < max_iter ? h_ctr[CTR_LAST] : max_iter);
    info_host[1] = (long long)run;
    info_host[2] = (long long)h_ctr[CTR_ACTIVE];
    info_host[3] = (long long)run * (long long)n * g.ntiles;
  }
  return converged ? B2_OK : B2_ERR_CONVERGE;
}

}  // namespace

extern "C" size_t b2_eikonal_work_bytes(size_t ny, size_t nx, size_t nz, size_t n) {
  if (!sizes_ok(ny, nx, nz, n)) return 0;
  return work_bytes(make_geom(ny, nx, nz, 1.0, 1.0, 1.0), n);
}

extern "C" int b2_eikonal_tables(b2_ctx* ctx, const double* vel, size_t ny, size_t nx, size_t nz, double dy,
                                 double dx, double dz, const long long* idx_host, size_t n, size_t max_iter,
                                 double* table, void* work, long long* info_host, void* stream) {
  if (!ctx || !vel || !idx_host || !table || !work) return B2_ERR_ARG;
  if (!sizes_ok(ny, nx, nz, n) || max_iter == 0) return B2_ERR_ARG;
  for (double h : {dy, dx, dz})
    if (!(h > 0.0) || !isfinite(h)) return B2_ERR_ARG;
  const size_t dims[3] = {ny, nx, nz};
  for (size_t p = 0; p < n; ++p)
    for (int a = 0; a < 3; ++a)
      if (idx_host[3 * p + a] < 0 || (size_t)idx_host[3 * p + a] >= dims[a]) return B2_ERR_ARG;
  const Geom g = make_geom(ny, nx, nz, dy, dx, dz);
  unsigned char* w = static_cast<unsigned char*>(work);
  const cudaStream_t st = (cudaStream_t)stream;
  return ny > 1 ? solve<3>(g, vel, idx_host, n, max_iter, table, w, info_host, st)
                : solve<2>(g, vel, idx_host, n, max_iter, table, w, info_host, st);
}
