// b2_xchg.cuh -- device side of the peer-memory exchange of the (D+2)^2 fp64 statistic (p2p.cu, gram_tc.cu, solve.cu).
//
// Every rank owns one exchange buffer that all peers have mapped (CUDA IPC between processes, plain peer access inside
// one process):
//     double slot[2 parities][kMaxRanks][kMaxS * kMaxS]      slot[e & 1][r] = rank r's partial S of exchange e
//     u32    flag[kMaxRanks]                                 flag[r] = last exchange whose slot r is complete here
//     u32    ticket (word 32), status (word 48)
// A producer stores its partial into slot[e & 1][rank] of EVERY buffer (st.global on peer pointers over
// NVLink / NVSwitch), fences at system scope and then writes e into flag[rank] of every buffer; a consumer waits until all
// flags of its OWN buffer carry e and sums the slots in rank order (bit-identical on every rank).  Slots are double
// buffered by parity: a rank can be at most one exchange ahead of a peer (its next wait needs that peer's next flag).
#pragma once
#include "b2_internal.cuh"
#include "b2_ptx.cuh"

namespace b2 {

struct PeerPtrs { double* p[kMaxRanks]; };

constexpr int kXchgTicketWord = 32;
constexpr int kXchgStatusWord = 48;

__host__ __device__ __forceinline__ unsigned int* xchg_flags(double* buf) {
  return reinterpret_cast<unsigned int*>(buf + kXchgDataDoubles);
}
__host__ __device__ __forceinline__ size_t xchg_slot_offset(unsigned int epoch, int rank) {
  return ((size_t)(epoch & 1u) * kMaxRanks + rank) * kXchgSlotDoubles;
}

// element idx of this rank's partial -> the same slot of every rank's buffer (own buffer included)
__device__ __forceinline__ void xchg_store_all(const PeerPtrs& peers, int n_ranks, size_t slot_off, int idx, double v) {
#pragma unroll 1
  for (int r = 0; r < n_ranks; ++r) peers.p[r][slot_off + idx] = v;
}

// Call by threads 0..n_ranks-1 of ONE block, after every store of this rank's partial has been fenced
// (__threadfence_system by the storing threads, then a block/grid level "all done" such as a ticket).
__device__ __forceinline__ void xchg_publish(const PeerPtrs& peers, int n_ranks, int rank, unsigned int epoch) {
  if ((int)threadIdx.x < n_ranks) {
    __threadfence_system();
    volatile unsigned int* f = xchg_flags(peers.p[threadIdx.x]) + rank;   // "rank has delivered exchange `epoch`"
    *f = epoch;
    __threadfence_system();
  }
}

// One thread: wait until every rank's slot of exchange `epoch` is complete in the own buffer.  Bounded by
// %globaltimer: a dead or very late peer yields `false` (and a status word the host reads), never a hung GPU.
__device__ __forceinline__ bool xchg_wait(double* own, int n_ranks, unsigned int epoch, unsigned long long timeout_ns) {
  volatile unsigned int* f = xchg_flags(own);
  const unsigned long long t0 = globaltimer_ns();
  for (int r = 0; r < n_ranks; ++r) {
    unsigned int spins = 0;
    while ((int)(f[r] - epoch) < 0) {                                   // exchange numbers are monotonic
      if ((++spins & 63u) == 0u) {
        if (globaltimer_ns() - t0 > timeout_ns) return false;
        __nanosleep(200);
      }
    }
  }
  __threadfence_system();
  return true;
}

// sum of the n slots of exchange `epoch` at element idx, in rank order (same order on every rank)
__device__ __forceinline__ double xchg_sum(const double* own, int n_ranks, unsigned int epoch, int idx) {
  const size_t base = (size_t)(epoch & 1u) * kMaxRanks * kXchgSlotDoubles;
  double s = 0.0;
  for (int r = 0; r < n_ranks; ++r) s += __ldcg(own + base + (size_t)r * kXchgSlotDoubles + idx);   // bypass L1
  return s;
}

}  // namespace b2
