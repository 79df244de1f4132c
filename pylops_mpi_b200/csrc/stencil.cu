// MPIFirstDerivative per-rank apply (reference:
// pylops_mpi/basicoperators/FirstDerivative.py:129-319).
//
// The operator is the banded matrix D (forward) or D^T (adjoint) acting along
// axis 0 of a [nrows_global x ncols] array; this rank owns rows
// [row0, row0+nrows_local) and receives up to 2 neighbour rows each side
// (the add_ghost_cells payload).  Every output row i is
//     y[i,:] = (sum_{k=-2..2} tap_k(i) * x[i+k,:]) * (1/sampling)
// with constant taps for interior rows and per-row taps for the first / last
// four GLOBAL rows (edge handling).  Adjoint taps are generated as the exact
// transpose of the forward taps, tap^T_k(i) = tap_{-k}(i+k), so <Dx,y> = <x,D^T y>
// holds by construction for every N, kind, order and edge flag.
//
// Fast path (HBM-bound, target >= 60 % of the HBM roofline): one thread owns a
// 16-byte column vector and a short chunk of rows held in a register window;
// every y element is written once with a streaming store.  Tuning:
// SHORT chunks win -- 4 rows per CTA keeps the
// concurrently running CTAs on a narrow band of whole rows (DRAM-page and L2
// friendly; the 2R overlap rows are L2 hits, DRAM traffic stays ~algorithmic),
// 64-row chunks (first design) reached 0.85 of the copy peak, 4-row chunks 1.04.
// Algorithmic bytes: 2*sizeof(T) per element.
#include "common.cuh"
#include "peer.cuh"

namespace {

constexpr int R = 2;           // max stencil radius
constexpr int NT = 2 * R + 1;  // taps per row
constexpr int SPECIAL = 4;     // rows at each global edge with their own taps
constexpr long long LONG_AXIS = 2000;   // an axis whose middle row is far from both edges

// one derivative operator: deriv 1 or 2, kind B2_FD_*, order 3 / 5 (centered first derivative only), edge, adjoint
struct FdOp { int deriv, kind, order, edge, adjoint; };

struct StencilParams {
  double interior[NT];
  double top[SPECIAL][NT];     // taps of global rows 0..3
  double bot[SPECIAL][NT];     // taps of global rows N-1, N-2, N-3, N-4
  double scale;                // 1/sampling
  long long nloc, ncols, row0, nglob;
  int n_lo, n_hi;
  long long batch_stride;      // elements between consecutive [nloc x ncols] problems (local axis-k derivatives)
  int nbatch;
};

// ---- halo rows over NVLink PEER MEMORY inside the stencil kernel (round 2) -----------------------------------
// The halo region of every rank's mailbox (peer.cuh) holds flags + 2 parities x 2 sides of halo rows.  The first
// column-tile CTAs of the kernel push this rank's boundary rows straight into the neighbours' regions (16-byte P2P
// stores) and publish a system-scope flag; only the CTAs that own the first / last row chunk wait for the
// neighbour's flag, and they are scheduled LAST, so the exchange hides behind the interior rows: ONE launch per
// apply, no NCCL call, no side stream (the reference does 2-4 add_ghost_cells exchanges per apply,
// FirstDerivative.py:221-247, 276-319).
struct HaloPeer {
  char* mine;        // this rank's halo region (local mapping)
  char* prev;        // rank-1's halo region (peer mapping) or nullptr
  char* next;        // rank+1's halo region or nullptr
  size_t cap;        // bytes per (parity, side) slot
  unsigned long long* seq;   // device: number of completed exchanges
  unsigned int* tickets;     // device: [0] push ticket, [1] edge ticket, [2] push-done marker
  int send_lo, send_hi;      // rows this rank sends to rank-1 / rank+1
};
__device__ __forceinline__ char* halo_slot(char* box, size_t cap, int par, int side) {
  return box + HALO_HDR + ((size_t)par * 2 + side) * cap;
}

// forward taps of global row i (offsets -2..2), before the 1/sampling scale
// second-derivative taps (MPISecondDerivative, basicoperators/SecondDerivative.py:125-257)
void fwd_taps2(long long i, long long N, int kind, int edge, double t[NT]) {
  if (kind == B2_FD_FORWARD) {            // y[i] = x[i] - 2 x[i+1] + x[i+2], i <= N-3      (:128-133)
    if (i <= N - 3) { t[R] = 1.0; t[R + 1] = -2.0; t[R + 2] = 1.0; }
  } else if (kind == B2_FD_BACKWARD) {    // y[i] = x[i-2] - 2 x[i-1] + x[i], i >= 2       (:160-165)
    if (i >= 2) { t[R - 2] = 1.0; t[R - 1] = -2.0; t[R] = 1.0; }
  } else {                                // centered                                      (:193-208)
    if (i >= 1 && i <= N - 2) { t[R - 1] = 1.0; t[R] = -2.0; t[R + 1] = 1.0; }
    else if (edge && N >= 3) {
      if (i == 0) { t[R] = 1.0; t[R + 1] = -2.0; t[R + 2] = 1.0; }
      if (i == N - 1) { t[R - 2] = 1.0; t[R - 1] = -2.0; t[R] = 1.0; }
    }
  }
}

void fwd_taps(long long i, long long N, int deriv, int kind, int order, int edge, double t[NT]) {
  for (int k = 0; k < NT; ++k) t[k] = 0.0;
  if (i < 0 || i >= N) return;
  if (deriv == 2) { fwd_taps2(i, N, kind, edge, t); return; }
  if (kind == B2_FD_FORWARD) {
    if (i <= N - 2) { t[R] = -1.0; t[R + 1] = 1.0; }
  } else if (kind == B2_FD_BACKWARD) {
    if (i >= 1) { t[R - 1] = -1.0; t[R] = 1.0; }
  } else if (order == 3) {
    if (i >= 1 && i <= N - 2) { t[R - 1] = -0.5; t[R + 1] = 0.5; }
    else if (edge && N >= 2) {
      if (i == 0) { t[R] += -1.0; t[R + 1] += 1.0; }
      if (i == N - 1) { t[R - 1] += -1.0; t[R] += 1.0; }
    }
  } else {  // centered, order 5
    if (i >= 2 && i <= N - 3) {
      t[R - 2] = 1.0 / 12.0; t[R - 1] = -2.0 / 3.0; t[R + 1] = 2.0 / 3.0; t[R + 2] = -1.0 / 12.0;
    } else if (edge) {
      // FirstDerivative.py:263-272: rank-0 writes y[0], y[1]; last rank writes y[-1], y[-2]
      // (later assignments overwrite earlier ones when N is tiny)
      double a[NT] = {0, 0, 0, 0, 0};
      bool set = false;
      if (i == 0 && N >= 2) { a[R] = -1.0; a[R + 1] = 1.0; set = true; }
      if (i == 1 && N >= 3) { for (int k = 0; k < NT; ++k) a[k] = 0; a[R - 1] = -0.5; a[R + 1] = 0.5; set = true; }
      if (i == N - 1 && N >= 2) { for (int k = 0; k < NT; ++k) a[k] = 0; a[R - 1] = -1.0; a[R] = 1.0; set = true; }
      if (i == N - 2 && N >= 3) { for (int k = 0; k < NT; ++k) a[k] = 0; a[R - 1] = -0.5; a[R + 1] = 0.5; set = true; }
      if (set) for (int k = 0; k < NT; ++k) t[k] = a[k];
    }
  }
}

void row_taps(long long i, long long N, const FdOp& op, double t[NT]) {
  if (!op.adjoint) { fwd_taps(i, N, op.deriv, op.kind, op.order, op.edge, t); return; }
  for (int k = -R; k <= R; ++k) {
    double f[NT];
    fwd_taps(i + k, N, op.deriv, op.kind, op.order, op.edge, f);   // zero outside [0, N)
    t[k + R] = f[-k + R];
  }
}

template <typename T>
__device__ __forceinline__ const T* row_ptr(const StencilParams& p, const T* x, const T* lo,
                                            const T* hi, long long r) {
  // r is a LOCAL row index in [-n_lo, nloc + n_hi); anything else -> nullptr
  if (r >= 0 && r < p.nloc) return x + r * p.ncols;
  if (r < 0) return (r >= -(long long)p.n_lo) ? lo + (p.n_lo + r) * p.ncols : nullptr;
  long long h = r - p.nloc;
  return (h < p.n_hi) ? hi + h * p.ncols : nullptr;
}

// row r of the extended block as a 16-byte vector; halo rows (written by a PEER GPU during this kernel in the
// peer-memory mode) go through the coherent load path, local rows through the read-only one
template <typename T>
__device__ __forceinline__ bool load_row(const StencilParams& p, const T* x, const T* lo, const T* hi, long long r,
                                         size_t coff, Vec16<T>& out) {
  if (r >= 0 && r < p.nloc) { out = load_vec(x + r * p.ncols + coff); return true; }
  const T* rp = row_ptr(p, x, lo, hi, r);
  if (!rp) return false;
  out = load_vec_coherent(rp + coff);
  return true;
}

__host__ __device__ __forceinline__ const double* special_taps(const StencilParams& p, long long gi) {
  if (gi < SPECIAL) return p.top[gi];
  if (gi >= p.nglob - SPECIAL) return p.bot[p.nglob - 1 - gi];
  return nullptr;
}

// -------------------------------------------------------------------------
// fast path: 16-byte column vectors, rolling window down a chunk of rows.
// MASK bit (k+R) set <=> interior tap k is non-zero (compile-time skip).
// -------------------------------------------------------------------------
constexpr int ST_ROWS = 4, ST_U = 4, ST_COLS = 128;   // rows per chunk, rows loaded per step, threads per CTA
template <typename T, int MASK, bool PEER>
__global__ void __launch_bounds__(ST_COLS)
stencil_vec_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ lo,
                   const T* __restrict__ hi, const __grid_constant__ StencilParams p, const HaloPeer hp) {
  constexpr int V = Vec16<T>::N;
  const long long ncv = p.ncols / V;
  // 1-D grid, column tile fastest: concurrently running CTAs cover whole rows
  const long long n_ct = (ncv + ST_COLS - 1) / ST_COLS;
  const long long ct = (long long)blockIdx.x % n_ct;
  long long rc = (long long)blockIdx.x / n_ct;
  x += (size_t)blockIdx.y * (size_t)p.batch_stride;     // batched local problems (blockIdx.y = 0 otherwise)
  y += (size_t)blockIdx.y * (size_t)p.batch_stride;
  const long long cv = ct * ST_COLS + threadIdx.x;
  [[maybe_unused]] bool edge_cta = false;
  [[maybe_unused]] unsigned long long seq = 0;
  [[maybe_unused]] long long n_edge = 0;
  if constexpr (PEER) {
    // chunk order: interior chunks first, the chunks next to the neighbours (0, n_rc-2, n_rc-1) LAST
    const long long n_rc = (p.nloc + ST_ROWS - 1) / ST_ROWS, j = rc;
    n_edge = n_rc < 3 ? n_rc : 3;
    if (j < n_rc - n_edge) rc = j + 1;
    else {
      const long long e = j - (n_rc - n_edge);
      rc = (e == 0) ? 0 : n_rc - n_edge + e;
      edge_cta = true;
    }
    seq = peer_next_seq(hp.seq);
    const int par = peer_parity(seq);
    if (j == 0) {
      // push my boundary rows into the neighbours' boxes (this CTA's column tile)
      if (cv < ncv) {
        const size_t cb = (size_t)cv * 16;
        if (hp.prev)
          for (int rr = 0; rr < hp.send_lo; ++rr)
            stg_stream16(halo_slot(hp.prev, hp.cap, par, 1) + (size_t)rr * p.ncols * sizeof(T) + cb,
                         ldg_stream16(x + (size_t)rr * p.ncols + (size_t)cv * V));
        if (hp.next)
          for (int rr = 0; rr < hp.send_hi; ++rr)
            stg_stream16(halo_slot(hp.next, hp.cap, par, 0) + (size_t)rr * p.ncols * sizeof(T) + cb,
                         ldg_stream16(x + (size_t)(p.nloc - hp.send_hi + rr) * p.ncols + (size_t)cv * V));
      }
      __threadfence_system();
      __syncthreads();
      if (threadIdx.x == 0) {
        const unsigned int t = atomicAdd(&hp.tickets[0], 1u);
        if (t == (unsigned int)n_ct - 1u) {      // every column tile of this rank is on its way: publish
          __threadfence_system();
          if (hp.prev) st_release_sys(&reinterpret_cast<HaloBox*>(hp.prev)->flag[par][1], seq);
          if (hp.next) st_release_sys(&reinterpret_cast<HaloBox*>(hp.next)->flag[par][0], seq);
          *reinterpret_cast<volatile unsigned int*>(&hp.tickets[2]) = 1u;
        }
      }
    }
    lo = reinterpret_cast<const T*>(halo_slot(hp.mine, hp.cap, par, 0));
    hi = reinterpret_cast<const T*>(halo_slot(hp.mine, hp.cap, par, 1));
  }
  const long long r0 = rc * ST_ROWS;
  const long long r1 = (r0 + ST_ROWS < p.nloc) ? r0 + ST_ROWS : p.nloc;
  if constexpr (PEER) {
    const int par = peer_parity(seq);
    const bool needs_lo = hp.prev && p.n_lo > 0 && r0 - R < 0;
    const bool needs_hi = hp.next && p.n_hi > 0 && r1 - 1 + R >= p.nloc;
    if (needs_lo || needs_hi) {
      if (threadIdx.x == 0) {
        const HaloBox* me = reinterpret_cast<const HaloBox*>(hp.mine);
        if (needs_lo) while (ld_acquire_sys(&me->flag[par][0]) < seq) { }
        if (needs_hi) while (ld_acquire_sys(&me->flag[par][1]) < seq) { }
      }
      __syncthreads();
    }
  }
  if (PEER ? false : (cv >= ncv)) return;
  const long long g0 = p.row0 + r0, g1 = p.row0 + r1;  // global rows [g0, g1)
  const bool has_special = (g0 < SPECIAL) || (g1 > p.nglob - SPECIAL);
  const size_t coff = (size_t)cv * V;
  const T scale = (T)p.scale;
  const bool do_scale = (p.scale != 1.0);

  if (PEER && cv >= ncv) {
    // inactive column lanes of a peer-mode CTA still take part in the barriers below
  } else if (!has_special) {
    T c[NT];
#pragma unroll
    for (int k = 0; k < NT; ++k) c[k] = (T)p.interior[k];
    // window w[j] holds local row (r - R + j) for the output row r being produced
    Vec16<T> w[NT + ST_U - 1];
#pragma unroll
    for (int j = 0; j < 2 * R; ++j) {
      if (!load_row(p, x, lo, hi, r0 - R + j, coff, w[j])) {
#pragma unroll
        for (int e = 0; e < V; ++e) w[j].v[e] = (T)0;
      }
    }
    for (long long r = r0; r < r1; r += ST_U) {
#pragma unroll
      for (int u = 0; u < ST_U; ++u) {
        if (!(r + u < r1 + R && load_row(p, x, lo, hi, r + u + R, coff, w[2 * R + u]))) {
#pragma unroll
          for (int e = 0; e < V; ++e) w[2 * R + u].v[e] = (T)0;
        }
      }
#pragma unroll
      for (int u = 0; u < ST_U; ++u) {
        if (r + u < r1) {
          Vec16<T> o;
#pragma unroll
          for (int e = 0; e < V; ++e) {
            T acc = (T)0;
#pragma unroll
            for (int k = 0; k < NT; ++k)
              if (MASK & (1 << k)) acc = fma(c[k], w[u + k].v[e], acc);
            o.v[e] = do_scale ? acc * scale : acc;
          }
          store_vec(y + (size_t)(r + u) * p.ncols + coff, o);
        }
      }
#pragma unroll
      for (int j = 0; j < 2 * R; ++j) w[j] = w[j + ST_U];
    }
  } else {
    // chunk touches a global edge: per-row taps, zero taps are skipped (never read)
    for (long long r = r0; r < r1; ++r) {
      const long long gi = p.row0 + r;
      const double* sp = special_taps(p, gi);
      Vec16<T> o;
#pragma unroll
      for (int e = 0; e < V; ++e) o.v[e] = (T)0;
#pragma unroll
      for (int k = 0; k < NT; ++k) {
        const double tk = sp ? sp[k] : p.interior[k];
        if (tk != 0.0) {
          Vec16<T> v;
          if (load_row(p, x, lo, hi, r + k - R, coff, v)) {
#pragma unroll
            for (int e = 0; e < V; ++e) o.v[e] = fma((T)tk, v.v[e], o.v[e]);
          }
        }
      }
      if (do_scale) {
#pragma unroll
        for (int e = 0; e < V; ++e) o.v[e] *= scale;
      }
      store_vec(y + (size_t)r * p.ncols + coff, o);
    }
  }
  if constexpr (PEER) {
    if (edge_cta) {
      // the last of the edge CTAs closes the exchange: it has seen BOTH neighbours' flags (so no rank can run
      // more than one exchange ahead of a neighbour: the two parities never collide) and this rank's push
      __syncthreads();
      if (threadIdx.x == 0) {
        const unsigned int t = atomicAdd(&hp.tickets[1], 1u);
        if (t == (unsigned int)(n_edge * n_ct) - 1u) {
          const int par = peer_parity(seq);
          const HaloBox* me = reinterpret_cast<const HaloBox*>(hp.mine);
          if (hp.prev) while (ld_acquire_sys(&me->flag[par][0]) < seq) { }
          if (hp.next) while (ld_acquire_sys(&me->flag[par][1]) < seq) { }
          while (*reinterpret_cast<volatile unsigned int*>(&hp.tickets[2]) == 0u) { }
          hp.tickets[0] = 0u;
          hp.tickets[1] = 0u;
          hp.tickets[2] = 0u;
          __threadfence();
          *reinterpret_cast<volatile unsigned long long*>(hp.seq) = seq;
        }
      }
    }
  }
}

// -------------------------------------------------------------------------
// generic path: one thread per output element (any ncols / alignment)
// -------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
stencil_generic_kernel(const T* x, T* y, const T* __restrict__ lo,
                       const T* __restrict__ hi, const __grid_constant__ StencilParams p) {
  const size_t per = (size_t)p.nloc * (size_t)p.ncols;
  const size_t total = per * (size_t)p.nbatch;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const T scale = (T)p.scale;
  const T* x0 = x;
  T* y0 = y;
  for (size_t gidx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; gidx < total; gidx += stride) {
    const size_t b = gidx / per, idx = gidx - b * per;
    x = x0 + b * (size_t)p.batch_stride;
    y = y0 + b * (size_t)p.batch_stride;
    const long long r = (long long)(idx / (size_t)p.ncols);
    const long long j = (long long)(idx - (size_t)r * (size_t)p.ncols);
    const long long gi = p.row0 + r;
    const double* sp = special_taps(p, gi);
    T acc = (T)0;
#pragma unroll
    for (int k = 0; k < NT; ++k) {
      const double tk = sp ? sp[k] : p.interior[k];
      if (tk != 0.0) {
        const T* rp = row_ptr(p, x, lo, hi, r + k - R);
        if (rp) acc = fma((T)tk, rp[j], acc);
      }
    }
    y[idx] = (p.scale != 1.0) ? acc * scale : acc;
  }
}

int interior_mask(const double t[NT]) {
  int m = 0;
  for (int k = 0; k < NT; ++k)
    if (t[k] != 0.0) m |= (1 << k);
  return m;
}

// PEER: the halo rows arrive through hp's peer boxes (lo / hi unused, one problem); otherwise from lo / hi, with
// p.nbatch problems along grid.y
template <typename T, bool PEER>
int launch_vec(const void* x, void* y, const void* lo, const void* hi, const StencilParams& p, const HaloPeer& hp,
               cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  const long long nblk = ((p.ncols / V + ST_COLS - 1) / ST_COLS) * ((p.nloc + ST_ROWS - 1) / ST_ROWS);
  if (nblk > 0x7fffffffLL) return B2_ERR_ARG;
  if (p.nbatch > 65535) return B2_ERR_ARG;
  const dim3 grid((unsigned)nblk, PEER ? 1u : (unsigned)p.nbatch);
#define B2_ST_LAUNCH(M) \
  stencil_vec_kernel<T, M, PEER><<<grid, ST_COLS, 0, st>>>((const T*)x, (T*)y, (const T*)lo, (const T*)hi, p, hp)
  switch (interior_mask(p.interior)) {
    case 0x0c: B2_ST_LAUNCH(0x0c); break;   // taps {0,+1}
    case 0x06: B2_ST_LAUNCH(0x06); break;   // taps {-1,0}
    case 0x0a: B2_ST_LAUNCH(0x0a); break;   // taps {-1,+1}
    case 0x1b: B2_ST_LAUNCH(0x1b); break;   // taps {-2,-1,+1,+2}
    default: B2_ST_LAUNCH(0x1f);
  }
#undef B2_ST_LAUNCH
  B2_LAUNCH_CHECK();
  return B2_OK;
}

template <typename T>
int launch_stencil(b2_ctx* ctx, const void* x, void* y, const void* lo, const void* hi,
                   const StencilParams& p, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  const bool vec_ok = (p.ncols % V == 0) && b2_aligned16(x) && b2_aligned16(y) &&
                      (!lo || b2_aligned16(lo)) && (!hi || b2_aligned16(hi)) &&
                      (p.ncols / V >= 8);
  if (vec_ok) return launch_vec<T, false>(x, y, lo, hi, p, HaloPeer{}, st);
  size_t total = (size_t)p.nloc * (size_t)p.ncols * (size_t)p.nbatch;
  size_t need = (total + 255) / 256;
  size_t cap = (size_t)ctx->sm_count * 8;
  int grid = (int)(need < cap ? need : cap);
  stencil_generic_kernel<T><<<grid, 256, 0, st>>>((const T*)x, (T*)y, (const T*)lo, (const T*)hi, p);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

// dtype F32 / F64 (complex data: the real dtype and twice the columns)
int launch_stencil(b2_ctx* ctx, const void* x, void* y, const void* lo, const void* hi, const StencilParams& p,
                   int dtype, cudaStream_t st) {
  return b2_dispatch_real(dtype, [&](auto t) { return launch_stencil<decltype(t)>(ctx, x, y, lo, hi, p, st); });
}

}  // namespace

// B2_ERR_UNSUPPORTED for an operator row_taps does not define (the entry points check deriv themselves)
static int fd_validate(const FdOp& op) {
  if (op.kind != B2_FD_FORWARD && op.kind != B2_FD_BACKWARD && op.kind != B2_FD_CENTERED) return B2_ERR_UNSUPPORTED;
  if (op.deriv == 1 && op.kind == B2_FD_CENTERED && op.order != 3 && op.order != 5) return B2_ERR_UNSUPPORTED;
  return B2_OK;
}

// how far below (*need_lo) and above (*need_hi) itself any row reads through op's non-zero taps (null: not
// written): on a long axis, rows 0..SPECIAL-1 and their mirror images have the edge taps, row SPECIAL the interior ones
static int fd_reach(const FdOp& op, int* need_lo, int* need_hi) {
  const int rc = fd_validate(op);
  if (rc) return rc;
  int lo = 0, hi = 0;
  for (long long i = 0; i <= SPECIAL; ++i)
    for (long long row : {i, LONG_AXIS - 1 - i}) {
      double t[NT];
      row_taps(row, LONG_AXIS, op, t);
      for (int k = 0; k < NT; ++k) {
        if (t[k] == 0.0) continue;
        if (R - k > lo) lo = R - k;
        if (k - R > hi) hi = k - R;
      }
    }
  if (need_lo) *need_lo = lo;
  if (need_hi) *need_hi = hi;
  return B2_OK;
}

static int b2_fd_build_params(StencilParams* p, int n_lo, int n_hi, size_t nrows_local, size_t ncols,
                              size_t row0, size_t nrows_global, const FdOp& op, double sampling) {
  const int rc = fd_validate(op);
  if (rc) return rc;
  if (row0 + nrows_local > nrows_global) return B2_ERR_ARG;
  const long long N = (long long)nrows_global;
  // interior taps = taps of a row far from both edges of a long axis
  row_taps(LONG_AXIS / 2, LONG_AXIS, op, p->interior);
  for (int s = 0; s < SPECIAL; ++s) {
    row_taps(s, N, op, p->top[s]);
    row_taps(N - 1 - s, N, op, p->bot[s]);
  }
  p->scale = (op.deriv == 2) ? 1.0 / (sampling * sampling) : 1.0 / sampling;
  p->batch_stride = 0;
  p->nbatch = 1;
  p->nloc = (long long)nrows_local;
  p->ncols = (long long)ncols;
  p->row0 = (long long)row0;
  p->nglob = N;
  p->n_lo = n_lo;
  p->n_hi = n_hi;
  return B2_OK;
}

// halo rows the block of p reads below (*lo) and above (*hi) itself: the non-zero taps of its first and last R
// rows, with the same per-row tap choice as the kernels (taps never reach outside the global array)
static void halo_reads(const StencilParams& p, int* lo, int* hi) {
  *lo = *hi = 0;
  auto scan = [&](long long r) {
    const double* t = special_taps(p, p.row0 + r);
    if (!t) t = p.interior;
    for (int k = 0; k < NT; ++k) {
      if (t[k] == 0.0) continue;
      const long long s = r + k - R;   // local row read
      if (s < 0 && -s > *lo) *lo = (int)-s;
      if (s >= p.nloc && s - p.nloc + 1 > *hi) *hi = (int)(s - p.nloc + 1);
    }
  };
  for (long long r = 0; r < p.nloc && r < R; ++r) scan(r);
  for (long long r = (p.nloc - R > R ? p.nloc - R : R); r < p.nloc; ++r) scan(r);
}

// one rank's row block with its halo rows: b2_first_derivative and b2_second_derivative
static int fd_block(b2_ctx* ctx, const void* x, void* y, const void* halo_lo, int n_lo, const void* halo_hi,
                    int n_hi, size_t nrows_local, size_t ncols, size_t row0, size_t nrows_global, const FdOp& op,
                    double sampling, int dtype, void* stream) {
  if (!ctx) return B2_ERR_ARG;
  if (nrows_local == 0 || ncols == 0) return B2_OK;
  if (!x || !y) return B2_ERR_ARG;
  if (n_lo < 0 || n_hi < 0 || n_lo > 8 || n_hi > 8) return B2_ERR_ARG;
  if (!halo_lo) n_lo = 0;
  if (!halo_hi) n_hi = 0;
  StencilParams p;
  const int rc = b2_fd_build_params(&p, n_lo, n_hi, nrows_local, ncols, row0, nrows_global, op, sampling);
  if (rc) return rc;
  int read_lo, read_hi;
  halo_reads(p, &read_lo, &read_hi);
  if (n_lo < read_lo || n_hi < read_hi) return B2_ERR_HALO;
  return launch_stencil(ctx, x, y, halo_lo, halo_hi, p, dtype, (cudaStream_t)stream);
}

extern "C" int b2_first_derivative_halo(int kind, int order, int adjoint, int* need_lo, int* need_hi) {
  int lo0, hi0, lo1, hi1;   // without / with edge handling: the wider reach is reported
  const int rc = fd_reach(FdOp{1, kind, order, 0, adjoint}, &lo0, &hi0);
  if (rc) return rc;
  fd_reach(FdOp{1, kind, order, 1, adjoint}, &lo1, &hi1);
  if (need_lo) *need_lo = lo0 > lo1 ? lo0 : lo1;
  if (need_hi) *need_hi = hi0 > hi1 ? hi0 : hi1;
  return B2_OK;
}

extern "C" int b2_first_derivative(b2_ctx* ctx, const void* x, void* y, const void* halo_lo, int n_lo,
                                   const void* halo_hi, int n_hi, size_t nrows_local, size_t ncols, size_t row0,
                                   size_t nrows_global, int kind, int order, int edge, double sampling, int adjoint,
                                   int dtype, void* stream) {
  return fd_block(ctx, x, y, halo_lo, n_lo, halo_hi, n_hi, nrows_local, ncols, row0, nrows_global,
                  FdOp{1, kind, order, edge, adjoint}, sampling, dtype, stream);
}

// ---- MPISecondDerivative per-rank apply (basicoperators/SecondDerivative.py:125-257) -----------------
extern "C" int b2_second_derivative_halo(int kind, int edge, int adjoint, int* need_lo, int* need_hi) {
  return fd_reach(FdOp{2, kind, 0, edge, adjoint}, need_lo, need_hi);
}

extern "C" int b2_second_derivative(b2_ctx* ctx, const void* x, void* y, const void* halo_lo, int n_lo,
                                    const void* halo_hi, int n_hi, size_t nrows_local, size_t ncols, size_t row0,
                                    size_t nrows_global, int kind, int edge, double sampling, int adjoint,
                                    int dtype, void* stream) {
  return fd_block(ctx, x, y, halo_lo, n_lo, halo_hi, n_hi, nrows_local, ncols, row0, nrows_global,
                  FdOp{2, kind, 0, edge, adjoint}, sampling, dtype, stream);
}

// One-launch distributed stencil: deriv = 1 (MPIFirstDerivative) or 2 (MPISecondDerivative); the halo rows
// travel through the halo regions of the mailboxes inside the kernel.  Collective over the ranks of the handle
// (same call sequence on every rank, one stream); every rank must own at least max(need_lo, need_hi) rows.
extern "C" int b2_derivative_peer(b2_ctx* ctx, b2_mailbox* h, const void* x, void* y, size_t nrows_local, size_t ncols,
                                  size_t row0, size_t nrows_global, int deriv, int kind, int order, int edge,
                                  double sampling, int adjoint, int dtype, void* stream) {
  if (!ctx || !h || !x || !y || (deriv != 1 && deriv != 2)) return B2_ERR_ARG;
  if (dtype != B2_F32 && dtype != B2_F64) return B2_ERR_DTYPE;
  const FdOp op{deriv, kind, order, edge, adjoint};
  int need_lo, need_hi;
  int rc = fd_reach(op, &need_lo, &need_hi);
  if (rc) return rc;
  const size_t esz = b2_dtype_size(dtype), V = 16 / esz;
  if ((long long)nrows_local < (need_lo > need_hi ? need_lo : need_hi)) return B2_ERR_HALO;
  if (ncols % V || ncols / V < 8 || !b2_aligned16(x) || !b2_aligned16(y)) return B2_ERR_ALIGN;
  if ((size_t)(need_lo > need_hi ? need_lo : need_hi) * ncols * esz > h->halo_cap) return B2_ERR_WORKSPACE;
  const bool has_prev = h->rank > 0, has_next = h->rank < h->size - 1;
  StencilParams p;
  rc = b2_fd_build_params(&p, has_prev ? need_lo : 0, has_next ? need_hi : 0, nrows_local, ncols, row0,
                          nrows_global, op, sampling);
  if (rc) return rc;
  HaloPeer hp;
  hp.mine = h->box[h->rank] + MB_HALO_OFF;
  hp.prev = has_prev ? h->box[h->rank - 1] + MB_HALO_OFF : nullptr;
  hp.next = has_next ? h->box[h->rank + 1] + MB_HALO_OFF : nullptr;
  hp.cap = h->halo_cap;
  hp.seq = &h->counters->seq[MB_SEQ_HALO];
  hp.tickets = h->counters->tickets;
  hp.send_lo = has_prev ? need_hi : 0;    // rank-1 needs my first need_hi rows as ITS hi halo
  hp.send_hi = has_next ? need_lo : 0;    // rank+1 needs my last need_lo rows as ITS lo halo
  cudaStream_t st = (cudaStream_t)stream;
  return b2_dispatch_real(dtype, [&](auto t) { return launch_vec<decltype(t), true>(x, y, nullptr, nullptr, p, hp, st); });
}

// ---- rank-local derivative along the MIDDLE axis of a C-ordered [n_outer][n_axis][n_inner] block ------
// (the non-partitioned directions of MPILaplacian / MPIGradient: Laplacian.py:97-126, Gradient.py:101-119
//  wrap a serial pylops First/SecondDerivative per rank; here the same stencil kernel runs batched)
extern "C" int b2_derivative_axis(b2_ctx* ctx, const void* x, void* y, size_t n_outer, size_t n_axis, size_t n_inner,
                                  int deriv, int kind, int order, int edge, double sampling, int adjoint, int dtype,
                                  void* stream) {
  if (!ctx || (deriv != 1 && deriv != 2)) return B2_ERR_ARG;
  if (n_outer == 0 || n_axis == 0 || n_inner == 0) return B2_OK;
  if (!x || !y) return B2_ERR_ARG;
  StencilParams p;
  int rc = b2_fd_build_params(&p, 0, 0, n_axis, n_inner, 0, n_axis, FdOp{deriv, kind, order, edge, adjoint},
                              sampling);
  if (rc) return rc;
  p.batch_stride = (long long)(n_axis * n_inner);
  cudaStream_t st = (cudaStream_t)stream;
  for (size_t done = 0; done < n_outer; done += 65535) {
    p.nbatch = (int)(n_outer - done < 65535 ? n_outer - done : 65535);
    const size_t off = done * n_axis * n_inner * b2_dtype_size(dtype);
    rc = launch_stencil(ctx, (const char*)x + off, (char*)y + off, nullptr, nullptr, p, dtype, st);
    if (rc) return rc;
  }
  return B2_OK;
}
