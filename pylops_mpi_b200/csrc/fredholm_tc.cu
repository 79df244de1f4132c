// MPIFredholm1 per-rank batched product on the Hopper tensor cores (wgmma; reference:
// pylops_mpi/signalprocessing/Fredholm1.py:119-132 forward `ncp.matmul(self.G, x)`, :147-170 adjoint
// `ncp.matmul(GT, x)` / `G.conj().transpose @ x`).
//
//   y[s] = op(G[s]) x[s],   s < nsl,   G[s]: nx x ny,  x[s]: (ny | nx) x nz,  float32 or complex64.
//
// float32-class accuracy on fp16 tensor cores ("fp16x2" split, an error-compensated split GEMM after Ootomo & Yokota):
// every fp32 number v is written as v*2^e = hi + lo*2^-11 with fp16 hi = rn(v 2^e), lo = rn((v 2^e - hi) 2^11)
// (22 significant bits; e = power-of-two scale per output row of op(G[s]) and per column of x[s], so that the largest
// element sits just below 2^15 -- undone exactly in the epilogue), and
//   a*b ~= hi_a hi_b + (hi_a lo_b + lo_a hi_b) 2^-11                  (dropped term <= 2^-22 |a||b|)
// is three tensor-core products on two planes per operand (the A planes take the 4 bytes/element of the float32
// original).  The tensor core's fp32 accumulate is lossier than an FMA chain (the error grows with the number of
// accumulator updates), so the leading term hi_a hi_b and the two correction terms go to TWO register accumulators
// that the epilogue adds (the corrections scaled by 2^-11): only K/16 updates touch the large accumulator instead of
// 3K/16.  Each operand tile is staged once per k-block and used by up to two of the three MMAs, so the L2->SMEM
// traffic per MMA is 2/3 that of a plain 128x128 fp16 GEMM tile.
//
// complex64 as one REAL product: G[s] viewed as floats is the real matrix A (nx x 2ny, columns = re,im
// interleaved); with X' (2ny x 2nz) built from x as
//      X'[2k  ,2z] =  re x[k,z]   X'[2k  ,2z+1] = im x[k,z]
//      X'[2k+1,2z] = -im x[k,z]   X'[2k+1,2z+1] = re x[k,z]
// A X' (nx x 2nz) IS the interleaved complex64 result.  Same flops as the complex product (8 nx ny nz).
//
// Operator state vs per-apply data: G is operator state -> its planes and row scales (and those of G^H, the
// reference's `saveGt`) are built ONCE at plan creation; x changes every apply -> a pack kernel takes the column
// scales of x and builds the two fp16 planes of X'^T (K-major, so both MMA operands are the canonical "TN" form)
// right before the product.
//
// Product kernel: persistent CTAs with 128 x 128 output tiles, warpgroup 0 = TMA producer (3-D tensor maps
// [k', row, slice*npl+plane], 128B swizzle, OOB zero fill => arbitrary nx, ny, nz), warpgroups 1-2 = consumers
// (wgmma.m64n128k16, 64 rows each, the two accumulators in registers), whose epilogue stores straight to y and
// -- fused all-gather of Fredholm1.py:131-132 -- the same 8-byte stores into every peer GPU's IPC-mapped output.
#include <string.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"

using namespace tcptx;

namespace {

constexpr uint32_t BM = 128, BN = 128, BK = 64, WG_K = 16;
constexpr uint32_t NUM_THREADS = 384;   // producer warpgroup + 2 consumer warpgroups (64 output rows each)
constexpr uint32_t ZSTRIP = 32;         // columns of x per pack block
constexpr uint32_t NPL = 2;             // planes per operand (hi, lo)
constexpr uint32_t NQ = 3;              // tensor-core products per k-step
constexpr uint32_t TILE_BYTES = 128 * BK * 2;             // one plane tile (128 rows x 64 16-bit, 128B swizzle)
constexpr uint32_t STAGE_BYTES = 2 * NPL * TILE_BYTES;     // A planes, B planes
constexpr uint32_t STAGES = (192u * 1024u) / STAGE_BYTES;  // 192 KB operand ring: 3 stages
constexpr size_t SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 + 256;

struct PeerOut {
  float* p[8];
  int n;
};

__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// v * sa * sb for power-of-two scales sa (row of op(G)) and sb (column of x).  sa * sb is exact unless it leaves the
// normal range, which needs both scales < 1 or both > 1 (tiny or huge maxima on both sides, while the result itself
// can still be a normal float or zero); then the scale nearer 1 goes first, so that the intermediate lies between v
// and the result and, for a normal result, only the last product rounds.
__device__ __forceinline__ float unscale(float v, float sa, float sb) {
  const float p = sa * sb;
  if (p >= 0x1p-126f && p <= 0x1p127f) return v * p;
  const float lo = fminf(sa, sb), hi = fmaxf(sa, sb);
  return p < 1.f ? (v * hi) * lo : (v * lo) * hi;
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
fredholm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   float* __restrict__ Y, const PeerOut peers, const float* __restrict__ invA,
                   const float* __restrict__ invB, uint32_t nz, uint32_t zdiv, uint32_t nsl, uint32_t m,
                   uint32_t n, uint32_t kpad, int vec_ok) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const uint32_t wg = threadIdx.x >> 7;
  const uint32_t num_m = (m + BM - 1) / BM, num_n = (n + BN - 1) / BN;
  const uint32_t num_tiles = nsl * num_m * num_n;
  const uint32_t num_kb = (kpad + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (uint32_t s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);     // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      bool dep_ready = false;     // the B planes are written by the pack kernel launched just before (PDL)
      for (uint32_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const uint32_t n_blk = tile % num_n, m_blk = (tile / num_n) % num_m, s = tile / (num_n * num_m);
        for (uint32_t kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + NPL * TILE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
#pragma unroll
          for (uint32_t p = 0; p < NPL; ++p)      // operator state: independent of the pack kernel
            tma_load_3d(sa + p * TILE_BYTES, &tmA, &full_bar[stage], (int32_t)(kb * BK), (int32_t)(m_blk * BM),
                        (int32_t)(s * NPL + p));
          if (!dep_ready) { grid_dep_wait(); dep_ready = true; }
#pragma unroll
          for (uint32_t p = 0; p < NPL; ++p)
            tma_load_3d(sb + p * TILE_BYTES, &tmB, &full_bar[stage], (int32_t)(kb * BK), (int32_t)(n_blk * BN),
                        (int32_t)(s * NPL + p));
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma into two accumulators, epilogue -> y (+ peers over NVLink) ===========
  setmaxnreg_inc<232>();
  const uint32_t cw = wg - 1;                       // rows [64 cw, 64 cw + 64) of the tile
  const uint32_t t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  const bool releaser = (t == 0);
  // small terms first; the LAST product of the list is the leading term (main accumulator)
  //   (hi,lo) (lo,hi) | (hi,hi)
  constexpr uint32_t pa[NQ] = {0u, 1u, 0u};
  constexpr uint32_t pb[NQ] = {1u, 0u, 0u};
  uint32_t stage = 0, phase = 0;
  float acc[BN / 2], sml[BN / 2];
  grid_dep_wait();     // y and the scales of x may only be touched once the previous kernel is done
  for (uint32_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const uint32_t n_blk = tile % num_n, m_blk = (tile / num_n) % num_m, s = tile / (num_n * num_m);
    uint32_t prev = STAGES;
    for (uint32_t kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + cw * 64 * 128;
      const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES) + NPL * TILE_BYTES;
      fence_regs(acc);
      fence_regs(sml);
      wgmma_fence();
#pragma unroll
      for (uint32_t kk = 0; kk < BK / WG_K; ++kk) {
#pragma unroll
        for (uint32_t q = 0; q < NQ; ++q) {
          // K-major, 128B swizzle: 8-row groups 1024 B apart, k advances 32 B inside the swizzle row
          const uint64_t adesc = make_smem_desc(sa + pa[q] * TILE_BYTES + kk * WG_K * 2, 16, 1024);
          const uint64_t bdesc = make_smem_desc(sb + pb[q] * TILE_BYTES + kk * WG_K * 2, 16, 1024);
          if (q == NQ - 1) wgmma_m64n128k16_f16<0, 0>(acc, adesc, bdesc, (kb | kk) != 0 ? 1 : 0);
          else wgmma_m64n128k16_f16<0, 0>(sml, adesc, bdesc, (kb | kk | q) != 0 ? 1 : 0);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                              // the previous k-block's MMAs are done: release its stage
      fence_regs(acc);
      fence_regs(sml);
      if (releaser && prev != STAGES) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    fence_regs(sml);
    if (releaser && prev != STAGES) mbar_arrive(&empty_bar[prev]);

    const uint32_t row0 = m_blk * BM + cw * 64 + warp * 16 + (lane >> 2);
    const uint32_t colb = n_blk * BN + 2 * (lane & 3);
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
      const uint32_t row = row0 + 8 * h;
      if (row >= m) continue;
      const size_t roff = ((size_t)s * m + row) * n;
      const float sa_inv = invA[(size_t)s * m + row];   // per output row
#pragma unroll
      for (uint32_t j = 0; j < BN / 8; ++j) {
        const uint32_t col = colb + 8 * j;
        if (col >= n) continue;
        // undo the power-of-two operand scales (exact: per output row of op(G), per column of x) and the 2^11
        // of the correction terms; complex columns (re, im) share a scale
        const float* sb_inv = invB + (size_t)s * nz;
        const float c0 = __ldg(sb_inv + col / zdiv);
        const float c1 = (col + 1 < n) ? __ldg(sb_inv + (col + 1) / zdiv) : 0.f;
        float2 o;
        o.x = unscale(fmaf(sml[4 * j + 2 * h], 1.f / 2048.f, acc[4 * j + 2 * h]), sa_inv, c0);
        o.y = unscale(fmaf(sml[4 * j + 2 * h + 1], 1.f / 2048.f, acc[4 * j + 2 * h + 1]), sa_inv, c1);
        const size_t off = roff + col;
        if (vec_ok && col + 1 < n) {
          *reinterpret_cast<float2*>(Y + off) = o;
          for (int d = 0; d < peers.n; ++d) *reinterpret_cast<float2*>(peers.p[d] + off) = o;
        } else {
          Y[off] = o.x;
          for (int d = 0; d < peers.n; ++d) peers.p[d][off] = o.x;
          if (col + 1 < n) {
            Y[off + 1] = o.y;
            for (int d = 0; d < peers.n; ++d) peers.p[d][off + 1] = o.y;
          }
        }
      }
    }
  }
}

// ---- operand splits (16-bit planes stored as raw ushort) ---------------------------------------------------
struct Split { unsigned short p[NPL]; };

__device__ __forceinline__ Split split(float v, float scale) {
  Split r;
  const float vs = v * scale;                      // |vs| < 2^15: no fp16 overflow
  const __half h0 = __float2half_rn(vs);
  r.p[0] = __half_as_ushort(h0);
  r.p[1] = __half_as_ushort(__float2half_rn((vs - __half2float(h0)) * 2048.f));
  return r;
}
__device__ __forceinline__ unsigned short neg16(unsigned short h) { return h ^ 0x8000u; }   // fp16: sign bit

// power-of-two scale that puts amax just below 2^15 (exponent clamped so scale and 1/scale stay normal floats; every
// finite float32 amax >= 2^-112 gets its exact scale, the largest ones need e = -113)
__device__ __forceinline__ void pow2_scale(float amax, float* scale, float* inv) {
  int ex = 0;
  if (amax > 0.f && amax < INFINITY) frexpf(amax, &ex);      // amax = f * 2^ex, f in [0.5, 1)
  else ex = 15;
  int e = 15 - ex;
  e = e > 126 ? 126 : (e < -126 ? -126 : e);
  *scale = ldexpf(1.f, e);
  *inv = ldexpf(1.f, -e);
}

__device__ __forceinline__ float block_max(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < nw; ++i) r = fmaxf(r, red[i]);
  __syncthreads();
  return r;
}

// power-of-two scale of every output ROW of op(G[s]) (operator state, once per plan and direction):
//   dir 0: row i of G[s] (contiguous);  dir 1: row j of G[s]^H = column j of G[s]
__global__ void __launch_bounds__(128) row_scale_kernel(const float* __restrict__ G, size_t nx, size_t ny, int cx, int dir,
                                                         float* scA, float* invA) {
  __shared__ float red[4];
  const size_t rows = dir == 0 ? nx : ny, inner = dir == 0 ? ny : nx;
  const size_t s = blockIdx.x / rows, r = blockIdx.x % rows;
  const size_t mul = cx ? 2 : 1;
  const float* g = G + s * nx * ny * mul;
  float am = 0.f;
  for (size_t q = threadIdx.x; q < inner * mul; q += blockDim.x) {
    const size_t e = q / mul, c = q % mul;
    const size_t idx = dir == 0 ? (r * ny + e) : (e * ny + r);
    am = fmaxf(am, fabsf(g[idx * mul + c]));
  }
  am = block_max(am, red);
  if (threadIdx.x == 0) pow2_scale(am, &scA[blockIdx.x], &invA[blockIdx.x]);
}

// operator state, once per plan: planes[s][p][r][c'] (c' < kpad, zero padded) of op(G[s]) as a real matrix.
//   dir 0:  r = i (nx rows),  c' = cx ? 2j+cc : j   <- G[s][i][j]            (cc: 0 = re, 1 = im)
//   dir 1:  r = j (ny rows),  c' = cx ? 2i+cc : i   <- conj(G[s][i][j])      (G^H)
__global__ void pack_g_kernel(const float* __restrict__ G, unsigned short* __restrict__ out, const float* __restrict__ scA,
                              size_t nsl, size_t nx, size_t ny, int cx, int dir, size_t rows, size_t kpad) {
  const size_t total = nsl * rows * kpad;
  const size_t kp = (dir == 0 ? ny : nx) * (cx ? 2 : 1);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t c = e % kpad, r = (e / kpad) % rows, s = e / (kpad * rows);
    float v = 0.f;
    if (c < kp) {
      const size_t inner = cx ? c / 2 : c;
      const int cc = cx ? (int)(c & 1) : 0;
      const size_t i = dir == 0 ? r : inner, j = dir == 0 ? inner : r;
      const size_t idx = (s * nx + i) * ny + j;
      v = cx ? G[2 * idx + cc] : G[idx];
      if (dir == 1 && cc == 1) v = -v;
    }
    const Split sp = split(v, scA[s * rows + r]);
    const size_t base = ((s * NPL) * rows + r) * kpad + c;
#pragma unroll
    for (uint32_t p = 0; p < NPL; ++p) out[base + (size_t)p * rows * kpad] = sp.p[p];
  }
}

// per apply: planes of X'^T,  BT[s][p][n'][k'] (k' < kpad; columns in [kp, kpad) are written as zeros)
//   complex: n' = 2z+d, k' = 2k+c:  (c,d) = (0,0) re, (1,0) -im, (0,1) im, (1,1) re
//   real   : n' = z,    k' = k
// Plane p of the splits of x[kb .. kb+3][z], packed as both pack kernels store it along k': complex x gives row 2z
// in r0 ((re, -im) pairs) and row 2z+1 in r1 ((im, re) pairs); real x gives row z in r0.x, r0.y and reads no im.
// The kernels keep the address arithmetic and the stores: moved in here, they compile to different, larger code.
template <bool CX>
__device__ __forceinline__ void plane_words(const Split (&re)[4], const Split (&im)[4], uint32_t p, uint4& r0, uint4& r1) {
  if (CX) {
    r0.x = re[0].p[p] | ((uint32_t)neg16(im[0].p[p]) << 16);  r1.x = im[0].p[p] | ((uint32_t)re[0].p[p] << 16);
    r0.y = re[1].p[p] | ((uint32_t)neg16(im[1].p[p]) << 16);  r1.y = im[1].p[p] | ((uint32_t)re[1].p[p] << 16);
    r0.z = re[2].p[p] | ((uint32_t)neg16(im[2].p[p]) << 16);  r1.z = im[2].p[p] | ((uint32_t)re[2].p[p] << 16);
    r0.w = re[3].p[p] | ((uint32_t)neg16(im[3].p[p]) << 16);  r1.w = im[3].p[p] | ((uint32_t)re[3].p[p] << 16);
  } else {
    r0.x = re[0].p[p] | ((uint32_t)re[1].p[p] << 16);
    r0.y = re[2].p[p] | ((uint32_t)re[3].p[p] << 16);
  }
}

// One 1024-thread block per (32-column strip of x, slice, 128-row tile of k): first takes every COLUMN's amax over
// all k (power-of-two scale per column, its inverse goes to invB for the epilogue), then the 128 x 32 tile is
// transposed through shared memory and written as 16-byte (complex) / 8-byte (real) vectors along k'.
constexpr uint32_t PK_THREADS = 1024, PK_ROWS = 128;
template <bool CX>
__global__ void __launch_bounds__(PK_THREADS)
pack_x_kernel(const float* __restrict__ x, unsigned short* __restrict__ BT, float* __restrict__ invB, uint32_t K,
              uint32_t nz, uint32_t nrows, uint32_t kpad) {
  __shared__ float2 tile[PK_ROWS][33];
  __shared__ float colmax[32][33];
  __shared__ float scale_s[32];
  grid_dep_launch();               // PDL: the product kernel may start its prologue / A loads now
  const uint32_t s = blockIdx.y, z0 = blockIdx.x * ZSTRIP;
  const uint32_t tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* xs = x + (size_t)s * K * nz * (CX ? 2 : 1);
  {
    float am = 0.f;
    const uint32_t z = z0 + tx;
    if (z < nz)
      for (uint32_t k = ty; k < K; k += 32) {
        if (CX) {
          const float2 v = reinterpret_cast<const float2*>(xs)[(size_t)k * nz + z];
          am = fmaxf(am, fmaxf(fabsf(v.x), fabsf(v.y)));
        } else {
          am = fmaxf(am, fabsf(xs[(size_t)k * nz + z]));
        }
      }
    colmax[ty][tx] = am;
    __syncthreads();
    if (ty == 0) {
      float m = colmax[0][tx];
      for (int i = 1; i < 32; ++i) m = fmaxf(m, colmax[i][tx]);
      float sc, inv;
      pow2_scale(m, &sc, &inv);
      scale_s[tx] = sc;
      if (z < nz && blockIdx.z == 0) invB[(size_t)s * nz + z] = inv;
    }
    __syncthreads();
  }
  const size_t plane = (size_t)nrows * kpad;
  unsigned short* base = BT + (size_t)s * NPL * plane;
  const uint32_t zz = threadIdx.x >> 5, kq = threadIdx.x & 31;     // write phase: one z, four consecutive k
  const float scale = scale_s[zz];
  // blockIdx.z selects ONE 128-row tile of k (the column scales above are recomputed by every k-block: a few L2
  // reads per thread, in exchange for twice the CTAs in flight on the config-5 shape)
  {
    const uint32_t k0 = blockIdx.z * PK_ROWS;
    for (uint32_t kk = ty; kk < PK_ROWS; kk += 32) {
      const uint32_t k = k0 + kk, z = z0 + tx;
      float2 v = make_float2(0.f, 0.f);
      if (k < K && z < nz) {
        if (CX) v = reinterpret_cast<const float2*>(xs)[(size_t)k * nz + z];
        else v.x = xs[(size_t)k * nz + z];
      }
      tile[kk][tx] = v;
    }
    __syncthreads();
    const uint32_t z = z0 + zz, kb = k0 + 4 * kq;
    if (z < nz && kb * (CX ? 2 : 1) < kpad) {
      Split re[4], im[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 v = tile[4 * kq + j][zz];
        re[j] = split(v.x, scale);
        if (CX) im[j] = split(v.y, scale);
      }
      #pragma unroll
      for (uint32_t p = 0; p < NPL; ++p) {
        unsigned short* q = base + p * plane;
        uint4 r0, r1;
        plane_words<CX>(re, im, p, r0, r1);
        if (CX) {
          *reinterpret_cast<uint4*>(q + (size_t)(2 * z) * kpad + 2 * kb) = r0;
          *reinterpret_cast<uint4*>(q + (size_t)(2 * z + 1) * kpad + 2 * kb) = r1;
        } else {
          *reinterpret_cast<uint2*>(q + (size_t)z * kpad + kb) = make_uint2(r0.x, r0.y);
        }
      }
    }
    __syncthreads();
  }
}

// Single-pass variant for short contractions (k' columns covered by <= PS_K values of k: config 5 has K = 256):
// one 256-thread block per (16-column strip of x, slice) reads its whole K x 16 strip ONCE -- 16 independent loads
// per thread in flight -- into shared memory, takes the column scales from the values it already holds and writes
// the planes.  Versus the generic kernel above: no second read of x, a quarter of the threads per block (faster
// block launch), 256 blocks for config 5.  Shared tile columns are rotated by k/4 so that both the row-wise fill
// and the 4-consecutive-k reads of the write phase are bank-conflict free.
constexpr uint32_t PS_THREADS = 256, PS_K = 256, PS_Z = 16;
template <bool CX>
__global__ void __launch_bounds__(PS_THREADS)
pack_x_small_kernel(const float* __restrict__ x, unsigned short* __restrict__ BT, float* __restrict__ invB, uint32_t K,
                    uint32_t nz, uint32_t nrows, uint32_t kpad) {
  __shared__ float2 tile[PS_K][PS_Z];
  __shared__ float colmax[PS_THREADS / PS_Z][PS_Z + 1];
  __shared__ float scale_s[PS_Z];
  grid_dep_launch();               // PDL: the product kernel may start its prologue / A loads now
  const uint32_t s = blockIdx.y, z0 = blockIdx.x * PS_Z;
  const uint32_t tx = threadIdx.x & (PS_Z - 1), ty = threadIdx.x / PS_Z;
  const float* xs = x + (size_t)s * K * nz * (CX ? 2 : 1);
  {
    const uint32_t z = z0 + tx;
    float2 v[PS_K / (PS_THREADS / PS_Z)];
#pragma unroll
    for (uint32_t i = 0; i < PS_K / (PS_THREADS / PS_Z); ++i) {
      const uint32_t k = ty + (PS_THREADS / PS_Z) * i;
      v[i] = make_float2(0.f, 0.f);
      if (k < K && z < nz) {
        if (CX) v[i] = reinterpret_cast<const float2*>(xs)[(size_t)k * nz + z];
        else v[i].x = xs[(size_t)k * nz + z];
      }
    }
    float am = 0.f;
#pragma unroll
    for (uint32_t i = 0; i < PS_K / (PS_THREADS / PS_Z); ++i) {
      const uint32_t k = ty + (PS_THREADS / PS_Z) * i;
      tile[k][(tx + (k >> 2)) & (PS_Z - 1)] = v[i];
      am = fmaxf(am, fmaxf(fabsf(v[i].x), fabsf(v[i].y)));
    }
    colmax[ty][tx] = am;
  }
  __syncthreads();
  if (threadIdx.x < PS_Z) {
    float m = colmax[0][threadIdx.x];
#pragma unroll
    for (uint32_t i = 1; i < PS_THREADS / PS_Z; ++i) m = fmaxf(m, colmax[i][threadIdx.x]);
    float sc, inv;
    pow2_scale(m, &sc, &inv);
    scale_s[threadIdx.x] = sc;
    if (z0 + threadIdx.x < nz) invB[(size_t)s * nz + z0 + threadIdx.x] = inv;
  }
  __syncthreads();
  const size_t plane = (size_t)nrows * kpad;
  unsigned short* base = BT + (size_t)s * NPL * plane;
#pragma unroll
  for (uint32_t it = 0; it < PS_Z * (PS_K / 4) / PS_THREADS; ++it) {
    const uint32_t item = threadIdx.x + PS_THREADS * it;
    const uint32_t kq = item & (PS_K / 4 - 1), zz = item / (PS_K / 4);
    const uint32_t z = z0 + zz, kb = 4 * kq;
    if (z >= nz || kb * (CX ? 2 : 1) >= kpad) continue;
    const float scale = scale_s[zz];
    Split re[4], im[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 v = tile[kb + j][(zz + kq) & (PS_Z - 1)];
      re[j] = split(v.x, scale);
      if (CX) im[j] = split(v.y, scale);
    }
    #pragma unroll
    for (uint32_t p = 0; p < NPL; ++p) {
      unsigned short* q = base + p * plane;
      uint4 r0, r1;
      plane_words<CX>(re, im, p, r0, r1);
      if (CX) {
        *reinterpret_cast<uint4*>(q + (size_t)(2 * z) * kpad + 2 * kb) = r0;
        *reinterpret_cast<uint4*>(q + (size_t)(2 * z + 1) * kpad + 2 * kb) = r1;
      } else {
        *reinterpret_cast<uint2*>(q + (size_t)z * kpad + kb) = make_uint2(r0.x, r0.y);
      }
    }
  }
}

// 3-D tensor map [k', row, slice*npl+plane] over fp16 planes; box = 64 k' (128 B, 128B swizzle) x box_rows x 1
int make_tmap3(CUtensorMap* tm, const void* base, uint64_t kpad, uint64_t rows, uint64_t nmat, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return B2_ERR_UNSUPPORTED;
  cuuint64_t gdim[3] = {kpad, rows, nmat};
  cuuint64_t gstr[2] = {kpad * 2, rows * kpad * 2};
  cuuint32_t box[3] = {BK, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base),
                  gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? B2_OK : B2_ERR_ARG;
}

size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

struct b2_fredholm_plan {
  b2_ctx* ctx;
  size_t nsl, nx, ny, nz;
  int cx;                       // complex64 (1) or float32 (0)
  // per direction d (0 forward, 1 adjoint): output rows m[d], contraction length kp[d] (real), padded kpad[d]
  size_t m[2], kp[2], kpad[2];
  unsigned short* A[2];         // planes of op(G): [nsl][npl][m][kpad]
  unsigned short* BT[2];        // planes of X'^T : [nsl][npl][n][kpad]   (per-apply workspace)
  float *scA[2], *invA[2], *invB;   // power-of-two scale per (slice, output row) of op(G) and its inverse (per
                                    // direction), inverse scale per (slice, column of x)
  uint32_t n, nstrips;          // output columns (real), 32-column strips of x
  CUtensorMap tmA[2], tmB[2];
};

extern "C" int b2_fredholm_plan_destroy(b2_fredholm_plan* pl) {
  if (!pl) return B2_OK;
  for (int d = 0; d < 2; ++d) {
    if (pl->A[d]) cudaFree(pl->A[d]);
    if (pl->BT[d]) cudaFree(pl->BT[d]);
  }
  for (int d = 0; d < 2; ++d) {
    if (pl->scA[d]) cudaFree(pl->scA[d]);
    if (pl->invA[d]) cudaFree(pl->invA[d]);
  }
  if (pl->invB) cudaFree(pl->invB);
  delete pl;
  return B2_OK;
}

extern "C" int b2_fredholm_plan_create(b2_ctx* ctx, const void* G, size_t nsl, size_t nx, size_t ny, size_t nz, int dtype,
                                       b2_fredholm_plan** out) {
  if (!ctx || !out || !G) return B2_ERR_ARG;
  if (dtype != B2_F32 && dtype != B2_C64) return B2_ERR_DTYPE;
  if (nsl == 0 || nx == 0 || ny == 0 || nz == 0) return B2_ERR_ARG;
  if (nsl * NPL > 0x7fffffffull || nsl > 65535 || nx > 0x3fffffffull || ny > 0x3fffffffull || nz > 0x3fffffffull) return B2_ERR_ARG;
  if (!b2_aligned16(G)) return B2_ERR_ALIGN;
  b2_fredholm_plan* pl = new b2_fredholm_plan();
  memset(pl, 0, sizeof(*pl));
  pl->ctx = ctx;
  pl->nsl = nsl; pl->nx = nx; pl->ny = ny; pl->nz = nz;
  pl->cx = dtype == B2_C64;
  const size_t mul = pl->cx ? 2 : 1;
  pl->n = (uint32_t)(nz * mul);
  pl->nstrips = (uint32_t)((nz + ZSTRIP - 1) / ZSTRIP);
  pl->m[0] = nx; pl->kp[0] = ny * mul;
  pl->m[1] = ny; pl->kp[1] = nx * mul;
  int rc = B2_OK;
  cudaError_t e = cudaMalloc((void**)&pl->invB, nsl * nz * sizeof(float));
  if (e != cudaSuccess) rc = (int)e;
  for (int d = 0; d < 2 && rc == B2_OK; ++d) {
    e = cudaMalloc((void**)&pl->scA[d], nsl * pl->m[d] * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc((void**)&pl->invA[d], nsl * pl->m[d] * sizeof(float));
    if (e != cudaSuccess) { rc = (int)e; break; }
    if (nsl * pl->m[d] > 0x7fffffffull) { rc = B2_ERR_ARG; break; }
    row_scale_kernel<<<(unsigned)(nsl * pl->m[d]), 128>>>((const float*)G, nx, ny, pl->cx, d, pl->scA[d], pl->invA[d]);
    e = cudaGetLastError();
    if (e != cudaSuccess) { rc = (int)e; break; }
    pl->kpad[d] = round_up(pl->kp[d], 8);
    const size_t a_elems = nsl * NPL * pl->m[d] * pl->kpad[d], b_elems = nsl * NPL * (size_t)pl->n * pl->kpad[d];
    e = cudaMalloc((void**)&pl->A[d], a_elems * 2);
    if (e == cudaSuccess) e = cudaMalloc((void**)&pl->BT[d], b_elems * 2);
    if (e == cudaSuccess) e = cudaMemset(pl->BT[d], 0, b_elems * 2);
    if (e != cudaSuccess) { rc = (int)e; break; }
    const size_t total = nsl * pl->m[d] * pl->kpad[d];
    size_t blocks = (total + 255) / 256;
    if (blocks > (size_t)ctx->sm_count * 32) blocks = (size_t)ctx->sm_count * 32;
    pack_g_kernel<<<(unsigned)blocks, 256>>>((const float*)G, pl->A[d], pl->scA[d], nsl, nx, ny, pl->cx, d, pl->m[d], pl->kpad[d]);
    e = cudaGetLastError();
    if (e != cudaSuccess) { rc = (int)e; break; }
    rc = make_tmap3(&pl->tmA[d], pl->A[d], pl->kpad[d], pl->m[d], nsl * NPL, BM);
    if (rc == B2_OK) rc = make_tmap3(&pl->tmB[d], pl->BT[d], pl->kpad[d], pl->n, nsl * NPL, BN);
  }
  if (rc == B2_OK) {
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) rc = (int)e;
  }
  if (rc != B2_OK) {
    b2_fredholm_plan_destroy(pl);
    return rc;
  }
  *out = pl;
  return B2_OK;
}

static int launch_product(b2_fredholm_plan* pl, int d, float* y, const PeerOut& po, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(fredholm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    attr_set = true;
  }
  const uint32_t m = (uint32_t)pl->m[d];
  const uint32_t num_tiles = (uint32_t)(pl->nsl * ((m + BM - 1) / BM) * ((pl->n + BN - 1) / BN));
  const uint32_t grid = num_tiles < (uint32_t)pl->ctx->sm_count ? num_tiles : (uint32_t)pl->ctx->sm_count;
  int vec_ok = ((((uintptr_t)y) & 7u) == 0 && (pl->n % 2) == 0) ? 1 : 0;     // 8-byte column pairs
  for (int i = 0; i < po.n; ++i)
    if (((uintptr_t)po.p[i]) & 7u) vec_ok = 0;
  // programmatic dependent launch: this kernel's prologue and its loads of the (static) A planes overlap the
  // tail of the pack kernel; griddepcontrol.wait guards everything that depends on the pack kernel's output
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  B2_CUDA(cudaLaunchKernelEx(&cfg, fredholm_tc_kernel, pl->tmA[d], pl->tmB[d], y, po, (const float*)pl->invA[d],
                             (const float*)pl->invB, (uint32_t)pl->nz, pl->cx ? 2u : 1u, (uint32_t)pl->nsl, m, pl->n,
                             (uint32_t)pl->kpad[d], vec_ok));
  return B2_OK;
}

// y[s] = op(G[s]) x[s] for all slices of the plan; peers_host (npeers <= 8, may be NULL/0): the same logical
// output position in peer GPUs' IPC-mapped buffers -- the epilogue stores every element there too (fused all-gather).
// Applies of one plan must be stream-ordered (they share the X' workspace).
extern "C" int b2_fredholm_apply(b2_fredholm_plan* pl, const void* x, void* y, void* const* peers_host, int npeers,
                                 int adjoint, void* stream) {
  if (!pl || !x || !y || npeers < 0 || npeers > 8 || (npeers && !peers_host)) return B2_ERR_ARG;
  const int d = adjoint ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  const uint32_t K = (uint32_t)(d == 0 ? pl->ny : pl->nx);
  const uint32_t nz = (uint32_t)pl->nz, kpad = (uint32_t)pl->kpad[d];
  const uint32_t kcover = kpad / (pl->cx ? 2u : 1u);          // k values whose k' columns exist (incl. padding)
  dim3 grid(pl->nstrips, (unsigned)pl->nsl, (kcover + PK_ROWS - 1) / PK_ROWS);
  if (grid.z > 65535u) return B2_ERR_ARG;
  const float* xf = (const float*)x;
  if (kcover <= PS_K) {
    dim3 gs((nz + PS_Z - 1) / PS_Z, (unsigned)pl->nsl);
    if (pl->cx) pack_x_small_kernel<true><<<gs, PS_THREADS, 0, st>>>(xf, pl->BT[d], pl->invB, K, nz, pl->n, kpad);
    else pack_x_small_kernel<false><<<gs, PS_THREADS, 0, st>>>(xf, pl->BT[d], pl->invB, K, nz, pl->n, kpad);
  } else {
    if (pl->cx) pack_x_kernel<true><<<grid, PK_THREADS, 0, st>>>(xf, pl->BT[d], pl->invB, K, nz, pl->n, kpad);
    else pack_x_kernel<false><<<grid, PK_THREADS, 0, st>>>(xf, pl->BT[d], pl->invB, K, nz, pl->n, kpad);
  }
  B2_LAUNCH_CHECK();
  PeerOut po;
  po.n = npeers;
  for (int i = 0; i < 8; ++i) po.p[i] = i < npeers ? (float*)peers_host[i] : nullptr;
  return launch_product(pl, d, (float*)y, po, st);
}
