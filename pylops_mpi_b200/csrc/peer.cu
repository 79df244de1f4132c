// One-shot collectives over NVLink PEER MEMORY (no NCCL call), on the mailboxes of peer.cuh, and the mailbox handle
// itself (b2_mailbox_*), which stencil.cu's fused halo exchange shares.
#include "peer.cuh"

// One-shot all-reduce of a few float64 scalars: every rank stores its partial values into its slot of every peer's
// scalar region, publishes its flag there, spins on its own region until all P flags of this sequence number arrived,
// and folds the P contributions in rank order (bit-identical on every rank).  This is the collective half of
// DistributedArray.dot / norm (DistributedArray.py:684-686, 714-757) and of the CGLS step scalars
// (cls_basic.py:389-401): latency ~ one NVLink round trip instead of an NCCL launch + ring/tree protocol.
namespace {
struct PeerPtrs {
  Slots* p[PEER_MAX];
};

__device__ __forceinline__ double ld_volatile(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// single CTA: the sequence number is read at entry and advanced at exit
__global__ void peer_allreduce_kernel(PeerPtrs pp, int rank, int P, double* __restrict__ vals, int k,
                                      unsigned long long* seq_dev, int op) {
  const unsigned long long seq = peer_next_seq(seq_dev);
  const int par = peer_parity(seq);
  const int t = threadIdx.x;
  if (t < P) {
    Slots* dst = pp.p[t];
    for (int j = 0; j < k; ++j) dst->data[par][rank][j] = vals[j];
    __threadfence_system();
    st_release_sys(&dst->flag[par][rank], seq);
  }
  __syncthreads();
  Slots* me = pp.p[rank];
  if (t < P) {
    while (ld_acquire_sys(&me->flag[par][t]) < seq) { }
  }
  __syncthreads();
  if (t < k) {
    double acc = ld_volatile(&me->data[par][0][t]);
    for (int r = 1; r < P; ++r) {
      const double v = ld_volatile(&me->data[par][r][t]);
      acc = (op == B2_SUM) ? acc + v : (op == B2_MAX ? fmax(acc, v) : fmin(acc, v));
    }
    vals[t] = acc;
  }
  __syncthreads();
  if (t == 0) *reinterpret_cast<volatile unsigned long long*>(seq_dev) = seq;
}
}  // namespace

extern "C" size_t b2_mailbox_bytes(size_t halo_cap) { return MB_HALO_OFF + HALO_HDR + 4 * halo_cap; }

// boxes_host[r]: rank r's box (b2_symm_alloc of b2_mailbox_bytes(halo_cap) bytes) as mapped in THIS process, own
// pointer for r == rank.  Zeroes the three headers of this rank's box and the counters.  Collective: every rank must
// have created its handle before any rank's first call on it (callers barrier on the host after b2_mailbox_create).
extern "C" int b2_mailbox_create(int rank, int size, void* const* boxes_host, size_t halo_cap, b2_mailbox** out) {
  if (!out || !boxes_host || size < 1 || size > PEER_MAX || rank < 0 || rank >= size || halo_cap == 0 ||
      (halo_cap % 16))
    return B2_ERR_ARG;
  b2_mailbox* h = new b2_mailbox();
  h->rank = rank;
  h->size = size;
  h->halo_cap = halo_cap;
  h->counters = nullptr;
  for (int r = 0; r < PEER_MAX; ++r) h->box[r] = r < size ? (char*)boxes_host[r] : nullptr;
  char* mine = h->box[rank];
  cudaError_t e = cudaMalloc((void**)&h->counters, sizeof(MailboxCounters));
  if (e == cudaSuccess) e = cudaMemset(h->counters, 0, sizeof(MailboxCounters));
  if (e == cudaSuccess) e = cudaMemset(mine, 0, sizeof(Slots));
  if (e == cudaSuccess) e = cudaMemset(mine + MB_VEC_OFF, 0, VEC_HDR_BYTES);
  if (e == cudaSuccess) e = cudaMemset(mine + MB_HALO_OFF, 0, HALO_HDR);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { if (h->counters) cudaFree(h->counters); delete h; return (int)e; }
  *out = h;
  return B2_OK;
}

extern "C" int b2_mailbox_destroy(b2_mailbox* h) {
  if (h && h->counters) cudaFree(h->counters);
  delete h;
  return B2_OK;
}

// in-place all-reduce of k <= 8 float64 values resident on the device
extern "C" int b2_peer_allreduce(b2_mailbox* h, double* vals_dev, int k, int op, void* stream) {
  if (!h || !vals_dev || k < 1 || k > VAL_MAX) return B2_ERR_ARG;
  if (op != B2_SUM && op != B2_MAX && op != B2_MIN) return B2_ERR_ARG;
  PeerPtrs pp;
  for (int r = 0; r < PEER_MAX; ++r) pp.p[r] = (Slots*)h->box[r];
  peer_allreduce_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(pp, h->rank, h->size, vals_dev, k,
                                                            &h->counters->seq[MB_SEQ_SCALAR], op);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

// =====================================================================================
// One-shot all-reduce (SUM) of a small/medium VECTOR over peer memory: the array Allreduce of
// MPIVStack._rmatvec (VStack.py:146-148) / block MatrixMult adjoint (MatrixMult.py:420-426) in the
// latency regime (config 2: n <= ~1e5 floats).  Every rank pushes its vector into its slot of every
// peer's vector region with 16-byte P2P stores, the last CTA to finish publishes a system-scope flag on all
// peers, every CTA then waits for the P flags in its OWN region and folds the P slots in rank order
// (bit-identical results on all ranks).
// =====================================================================================
namespace {
struct VecPtrs {
  char* p[PEER_MAX];
};
__device__ __forceinline__ char* vec_slot(char* base, int par, int src) {
  return base + VEC_HDR_BYTES + ((size_t)par * PEER_MAX + src) * VEC_SLOT_BYTES;
}

// The exchange both vector kernels make: every CTA pushes its share of this rank's data into this rank's slot of
// every peer's region (push(slot) once per peer), the LAST CTA to finish advances the sequence counter and publishes
// the flags, and every CTA waits for the P flags of this call in its own region.  Returns the parity.  No CTA can
// leave the wait before the counter has advanced: every flag depends on every rank's last CTA.
template <typename Push>
__device__ __forceinline__ int vec_exchange(const VecPtrs& pp, int rank, int P, unsigned long long* seq_dev,
                                            Push push) {
  const unsigned long long seq = peer_next_seq(seq_dev);
  const int par = peer_parity(seq);
  for (int d = 0; d < P; ++d) push(vec_slot(pp.p[d], par, rank));
  __threadfence_system();
  __syncthreads();
  VecBox* me = reinterpret_cast<VecBox*>(pp.p[rank]);
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&me->arrive[par], 1u);
    if (t == gridDim.x - 1) {           // last CTA: everything of this rank is on its way -> publish
      me->arrive[par] = 0u;
      *reinterpret_cast<volatile unsigned long long*>(seq_dev) = seq;
      __threadfence_system();
      for (int d = 0; d < P; ++d)
        st_release_sys(&reinterpret_cast<VecBox*>(pp.p[d])->flag[par][rank], seq);
    }
  }
  if (threadIdx.x < P) {
    while (ld_acquire_sys(&me->flag[par][threadIdx.x]) < seq) { }
  }
  __syncthreads();
  return par;
}

template <typename T>
__global__ void __launch_bounds__(256)
peer_allreduce_vec_kernel(VecPtrs pp, int rank, int P, T* __restrict__ buf, size_t n, unsigned long long* seq_dev) {
  constexpr int V = 16 / sizeof(T);
  const size_t nvec = n / V;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
  const int par = vec_exchange(pp, rank, P, seq_dev, [&](char* slot) {
    T* dst = reinterpret_cast<T*>(slot);
    for (size_t i = tid; i < nvec; i += nthr)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(buf)[i];
    for (size_t i = nvec * V + tid; i < n; i += nthr) dst[i] = buf[i];
  });
  for (size_t i = tid; i < n; i += nthr) {
    T acc = *reinterpret_cast<volatile const T*>(reinterpret_cast<const T*>(vec_slot(pp.p[rank], par, 0)) + i);
    for (int r = 1; r < P; ++r)
      acc += *reinterpret_cast<volatile const T*>(reinterpret_cast<const T*>(vec_slot(pp.p[rank], par, r)) + i);
    buf[i] = acc;
  }
}
}  // namespace

// One-shot ALL-GATHER(v) over the same regions: every rank pushes its chunk into its slot of every peer's
// region, publishes its flag, waits for the P flags in its own region and copies the P slots into the contiguous
// result (rank order).  Replaces ncclAllGather in the latency regime (<= 256 KB per rank): the gather of the model
// vector in MPIMatrixMult's M = 1 "32768-vec" apply, small BROADCAST rebuilds (Fredholm1 KATs) ...
struct GatherCounts {
  unsigned long long bytes[PEER_MAX];   // chunk size of every rank
  unsigned long long off[PEER_MAX];     // byte offset of every rank's chunk in the result
};
template <typename W>   // W = uint4 / uint32_t / uint16_t copy word
__global__ void __launch_bounds__(256)
peer_allgather_vec_kernel(VecPtrs pp, int rank, int P, const char* __restrict__ send, char* __restrict__ recv,
                          GatherCounts gc, unsigned long long* seq_dev) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
  const size_t nw = gc.bytes[rank] / sizeof(W);
  const int par = vec_exchange(pp, rank, P, seq_dev, [&](char* slot) {
    W* dst = reinterpret_cast<W*>(slot);
    for (size_t i = tid; i < nw; i += nthr) dst[i] = reinterpret_cast<const W*>(send)[i];
  });
  for (int r = 0; r < P; ++r) {
    const volatile W* src = reinterpret_cast<const volatile W*>(vec_slot(pp.p[rank], par, r));
    W* out = reinterpret_cast<W*>(recv + gc.off[r]);
    const size_t n = gc.bytes[r] / sizeof(W);
    if constexpr (sizeof(W) == 16) {
      for (size_t i = tid; i < n; i += nthr) {
        uint4 v;
        const volatile uint32_t* s32 = reinterpret_cast<const volatile uint32_t*>(src + i);
        v.x = s32[0]; v.y = s32[1]; v.z = s32[2]; v.w = s32[3];
        reinterpret_cast<uint4*>(out)[i] = v;
      }
    } else {
      for (size_t i = tid; i < n; i += nthr) out[i] = src[i];
    }
  }
}

static VecPtrs vec_ptrs(const b2_mailbox* h) {
  VecPtrs pp;
  for (int r = 0; r < PEER_MAX; ++r) pp.p[r] = h->box[r] ? h->box[r] + MB_VEC_OFF : nullptr;
  return pp;
}

extern "C" size_t b2_peer_vec_max_bytes(void) { return VEC_SLOT_BYTES; }

// in-place SUM all-reduce of n elements (n * sizeof <= b2_peer_vec_max_bytes()), dtype F32 / F64
extern "C" int b2_peer_vec_allreduce(b2_mailbox* h, void* buf_dev, size_t n, int dtype, void* stream) {
  if (!h || !buf_dev) return B2_ERR_ARG;
  if (n == 0) return B2_OK;
  const size_t esz = b2_dtype_size(dtype);
  if ((dtype != B2_F32 && dtype != B2_F64) || n * esz > VEC_SLOT_BYTES) return B2_ERR_ARG;
  if (!b2_aligned16(buf_dev)) return B2_ERR_ALIGN;
  // few CTAs: all of them spin on flags, so they must be co-resident (16 << the SM count)
  size_t work = (n * esz + 16 * 256 - 1) / (16 * 256);
  const unsigned grid = (unsigned)(work < 1 ? 1 : (work > 16 ? 16 : work));
  cudaStream_t st = (cudaStream_t)stream;
  const VecPtrs pp = vec_ptrs(h);
  unsigned long long* seq = &h->counters->seq[MB_SEQ_VEC];
  if (dtype == B2_F32)
    peer_allreduce_vec_kernel<float><<<grid, 256, 0, st>>>(pp, h->rank, h->size, (float*)buf_dev, n, seq);
  else
    peer_allreduce_vec_kernel<double><<<grid, 256, 0, st>>>(pp, h->rank, h->size, (double*)buf_dev, n, seq);
  B2_LAUNCH_CHECK();
  return B2_OK;
}


// recv = concatenation of every rank's counts_host[r] elements (rank order); every chunk <= b2_peer_vec_max_bytes()
extern "C" int b2_peer_vec_allgatherv(b2_mailbox* h, const void* send, void* recv, const size_t* counts_host, int dtype,
                                      void* stream) {
  if (!h || !recv || !counts_host) return B2_ERR_ARG;
  const size_t esz = b2_dtype_size(dtype);
  if (esz == 0) return B2_ERR_DTYPE;
  GatherCounts gc;
  size_t off = 0, maxb = 0;
  int align = 16;
  for (int r = 0; r < PEER_MAX; ++r) {
    const size_t b = r < h->size ? counts_host[r] * esz : 0;
    gc.bytes[r] = b;
    gc.off[r] = off;
    if (b > maxb) maxb = b;
    if (b % 16 || off % 16) align = (b % 4 || off % 4) ? ((align > 2) ? 2 : align) : ((align > 4) ? 4 : align);
    off += b;
  }
  if (maxb > VEC_SLOT_BYTES) return B2_ERR_ARG;
  if (off == 0) return B2_OK;
  if (gc.bytes[h->rank] && !send) return B2_ERR_ARG;
  if (align == 16 && ((send && !b2_aligned16(send)) || !b2_aligned16(recv))) align = 4;
  if (align == 4 && ((((uintptr_t)send) | ((uintptr_t)recv)) & 3u)) align = 2;
  if (align == 2 && (esz % 2)) return B2_ERR_ALIGN;
  size_t work = (maxb + 16 * 256 - 1) / (16 * 256);
  const unsigned grid = (unsigned)(work < 1 ? 1 : (work > 16 ? 16 : work));    // all CTAs spin on flags: keep them co-resident
  cudaStream_t st = (cudaStream_t)stream;
  const VecPtrs pp = vec_ptrs(h);
  unsigned long long* seq = &h->counters->seq[MB_SEQ_VEC];
  if (align == 16)
    peer_allgather_vec_kernel<uint4><<<grid, 256, 0, st>>>(pp, h->rank, h->size, (const char*)send, (char*)recv, gc, seq);
  else if (align == 4)
    peer_allgather_vec_kernel<uint32_t><<<grid, 256, 0, st>>>(pp, h->rank, h->size, (const char*)send, (char*)recv, gc, seq);
  else
    peer_allgather_vec_kernel<uint16_t><<<grid, 256, 0, st>>>(pp, h->rank, h->size, (const char*)send, (char*)recv, gc, seq);
  B2_LAUNCH_CHECK();
  return B2_OK;
}
