// Peer-memory mailboxes: the protocol that the one-shot collectives of peer.cu and the halo exchange inside the
// stencil kernel (stencil.cu) share.
//
// Every rank owns ONE box in IPC-mapped device memory and maps every peer's.  The box has one region per use, each
// 256-byte aligned:  [scalar Slots | vector box | halo box].  A call writes into the peers' boxes, publishes a
// sequence number with a system-scope release store to a flag in each peer's box, and waits with an acquire spin on
// the flags in its own box.  The sequence number of each use lives in device memory (read at entry, advanced once
// the call has seen every flag it waits for), so a call is a plain kernel launch that a CUDA graph can capture.
// Every region is double-buffered by the parity of that number: a rank can run at most one call ahead of its
// slowest peer, because call n + 1 cannot complete before every peer has entered it.
#pragma once
#include "common.cuh"

constexpr int PEER_MAX = 8;

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// the sequence number of the call being made (one past the last completed one) and the half of the region it uses
__device__ __forceinline__ unsigned long long peer_next_seq(const unsigned long long* seq_dev) {
  return *reinterpret_cast<const volatile unsigned long long*>(seq_dev) + 1ull;
}
__device__ __forceinline__ int peer_parity(unsigned long long seq) { return (int)(seq & 1ull); }

// ---- the box of one rank --------------------------------------------------------------------------------------
// scalar region: k <= 8 float64 values of every rank, then one flag per rank
constexpr int VAL_MAX = 8;
struct Slots {
  double data[2][PEER_MAX][VAL_MAX];
  unsigned long long flag[2][PEER_MAX];
};
// vector region: a 256-byte header, then one slot per (parity, source rank)
constexpr size_t VEC_SLOT_BYTES = 256 * 1024;
constexpr size_t VEC_HDR_BYTES = 256;
struct VecBox {
  unsigned long long flag[2][PEER_MAX];
  unsigned int arrive[2];   // CTAs of this rank's call that have pushed their share
  unsigned int pad[2];
};
static_assert(sizeof(VecBox) <= VEC_HDR_BYTES, "header too small");
// halo region: a 256-byte header, then one slot of cap bytes per (parity, side)
constexpr size_t HALO_HDR = 256;
struct HaloBox {
  unsigned long long flag[2][2];   // [parity][side]: side 0 = rows from rank-1, side 1 = rows from rank+1
};

constexpr size_t peer_round256(size_t b) { return (b + 255) / 256 * 256; }
constexpr size_t MB_VEC_OFF = peer_round256(sizeof(Slots));
constexpr size_t MB_VEC_BYTES = VEC_HDR_BYTES + 2 * PEER_MAX * VEC_SLOT_BYTES;
constexpr size_t MB_HALO_OFF = MB_VEC_OFF + peer_round256(MB_VEC_BYTES);

// sequence counters (device memory), one per use so that each keeps its own one-call-ahead bound
enum { MB_SEQ_SCALAR = 0, MB_SEQ_VEC = 1, MB_SEQ_HALO = 2 };
struct MailboxCounters {
  unsigned long long seq[3];
  unsigned int tickets[4];   // halo exchange: [0] push ticket, [1] edge ticket, [2] push-done marker
};

struct b2_mailbox {
  int rank, size;
  char* box[PEER_MAX];          // box[r]: rank r's box as mapped in this process (nullptr for r >= size)
  size_t halo_cap;              // bytes per (parity, side) slot of the halo region
  MailboxCounters* counters;    // device
};
