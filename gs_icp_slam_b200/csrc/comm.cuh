// comm.cuh — multi-GPU exchange layer of libgsicp_b200.so: one symmetric device segment per rank, mapped into every
// peer with CUDA IPC (NVLink peer access), and device-side flag protocols on top of it.
//
// The two hot paths exchange very little data, very often (SURVEY.md §8e): 28 doubles per LM reduction point, 48 bytes
// per visible Gaussian per mapper iteration.  A host-launched collective per exchange costs more than the kernels it
// separates (r1: two NCCL all-reduces and a Python callback per LM iteration), so the exchange happens INSIDE our kernels:
// a rank's block writes its partial sums straight into every peer's segment (st.global over NVLink), releases a
// sequence flag, and every block of every rank sums the world's slots in rank order — identical bits everywhere, no
// host hop, no second kernel.
//
// Segment layout (same on every rank):
//   [0, 4 KB)        stream-barrier flags        u64 bar_flag[kMaxRanks]        (written by peers)
//   [4 KB, 8 KB)     LM exchange flags           u64 lm_flag[2][kMaxRanks]      (parity, writer rank)
//   [8 KB, 24 KB)    LM exchange data            f64 lm_data[2][kMaxRanks][32]
//   [24 KB, ...)     heap                        render-moment accumulators [P][12] f32, merge staging
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "host_common.h"

namespace gsicp {

constexpr int kMaxRanks = 16;
constexpr size_t kCommBarOff = 0, kCommLmFlagOff = 4096, kCommLmDataOff = 8192, kCommHeapOff = 24576;
constexpr int kLmSlotDoubles = 32;
constexpr long long kCommPollBudget = 1ll << 28;  // flag polls before a kernel gives up (seconds)

struct CommView {  // passed by value to kernels; world == 1 means "no peers"
  int world = 1, rank = 0;
  char* seg[kMaxRanks] = {};  // seg[r]: rank r's segment as mapped in this process (seg[rank] = local)
  __host__ __device__ bool active() const { return world > 1; }
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ double ld_volatile_f64(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// Publish `count` (<= 32) doubles of this rank for exchange number `seq` into every rank's segment (own included).
// Called by ONE block; threads t < count write, thread 0 releases the flags.  `vals` is in shared memory.
__device__ __forceinline__ void comm_lm_publish(const CommView& c, unsigned long long seq, const double* vals, int count) {
  const int par = (int)(seq & 1ull);
  if ((int)threadIdx.x < count) {
    for (int r = 0; r < c.world; r++) {
      double* dst = reinterpret_cast<double*>(c.seg[r] + kCommLmDataOff) + ((size_t)par * kMaxRanks + c.rank) * kLmSlotDoubles;
      dst[threadIdx.x] = vals[threadIdx.x];
    }
    __threadfence_system();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int r = 0; r < c.world; r++) {
      unsigned long long* f = reinterpret_cast<unsigned long long*>(c.seg[r] + kCommLmFlagOff) + (size_t)par * kMaxRanks + c.rank;
      st_release_sys(f, seq);
    }
  }
}

// Wait until every rank has published exchange `seq`, then sum the slots in rank order into out[count] (shared memory).
// Called by every block; returns false when the poll budget ran out (a peer died).
__device__ __forceinline__ bool comm_lm_collect(const CommView& c, unsigned long long seq, double* out, int count) {
  __shared__ int s_ok;
  const int par = (int)(seq & 1ull);
  const char* loc = c.seg[c.rank];
  if (threadIdx.x == 0) {
    int ok = 1;
    for (int r = 0; r < c.world && ok; r++) {
      const unsigned long long* f = reinterpret_cast<const unsigned long long*>(loc + kCommLmFlagOff) + (size_t)par * kMaxRanks + r;
      long long polls = 0;
      while (ld_acquire_sys(f) < seq) {
        if (++polls > kCommPollBudget) {
          ok = 0;
          break;
        }
      }
    }
    s_ok = ok;
  }
  __syncthreads();
  if (s_ok && (int)threadIdx.x < count) {
    double r0 = 0.0;
    for (int r = 0; r < c.world; r++) {
      const double* src = reinterpret_cast<const double*>(loc + kCommLmDataOff) + ((size_t)par * kMaxRanks + r) * kLmSlotDoubles;
      r0 += ld_volatile_f64(src + threadIdx.x);
    }
    out[threadIdx.x] = r0;
  }
  __syncthreads();
  return s_ok != 0;
}
#endif  // __CUDACC__

}  // namespace gsicp

// Host-side object behind the opaque gsicp_comm of include/gsicp_b200.h
struct gsicp_comm {
  int world = 1, rank = 0;
  int device = 0;
  size_t bytes = 0;
  char* local = nullptr;
  char* peer[gsicp::kMaxRanks] = {};
  bool connected = false;
  bool local_only = false;         // test hook: all ranks in one process (gsicp_comm_connect_local)
  unsigned long long bar_seq = 0;  // stream-barrier sequence (host-side counter; identical call order on every rank)
  unsigned long long lm_seq = 0;   // last LM exchange sequence number handed out (host-side, identical on every rank)
  bool lm_resync = false;          // the last launch consumed a data-dependent number of exchanges: re-align with a barrier
  gsicp::Mapped<int> status;       // status.h[0]: a barrier kernel sets it when its poll budget ran out (a peer is gone)
  gsicp::CommView view() const {
    gsicp::CommView v;
    v.world = world;
    v.rank = rank;
    for (int r = 0; r < world && r < gsicp::kMaxRanks; r++) v.seg[r] = peer[r];
    return v;
  }
  size_t heap_bytes() const { return bytes > gsicp::kCommHeapOff ? bytes - gsicp::kCommHeapOff : 0; }
};

namespace gsicp {
// Enqueue a barrier over all ranks on `stream`: everything this rank enqueued before it is visible to the peers'
// kernels enqueued after THEIR matching barrier.
int comm_stream_barrier(gsicp_comm* c, cudaStream_t stream);
}  // namespace gsicp
