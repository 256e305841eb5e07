// gicp_reduce.cuh — pieces shared by the host-driven linearisation kernels of GICP (gicp.cu) and VGICP (vgicp.cu): the
// pose in both precisions and the deterministic 28-value block reduction.  Both translation units are compiled with
// -fmad=false.
#pragma once
#include "gicp_math.cuh"
#include "comm.cuh"
#include "host_common.h"

namespace gsicp {

constexpr int kRed = 28;       // 21 (upper triangle of H, row-major) + 6 (b) + 1 (error)
constexpr int kLinBlock = 128;

struct PoseD {  // pose in both precisions, passed by value
  double R[3][3], t[3];
  float Rf[3][3], tf[3];
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-level reduction of NV doubles per thread into partial[blockIdx][NV]; the last block to finish
// sums the partials in block order (deterministic) into out[NV].
//
// When `host_out` is non-null (single-GPU runs) the last block also publishes the sums into MAPPED PINNED host memory and
// then bumps a sequence word the host spins on: the result reaches the LM loop without a D2H memcpy or a
// cudaStreamSynchronize round trip (two driver calls and a thread wake-up per launch otherwise).
template <int NV>
__device__ __forceinline__ void block_reduce_finalize(double* v, double* __restrict__ partial, double* __restrict__ out,
                                                      unsigned int* __restrict__ counter, double* host_out = nullptr,
                                                      volatile unsigned long long* host_seq = nullptr,
                                                      unsigned long long seq = 0, CommView comm = CommView(),
                                                      unsigned long long xseq = 0) {
  __shared__ double s_red[kLinBlock / 32][NV];
  __shared__ double s_tot[NV];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; k++) {
    const double r = warp_sum_d(v[k]);
    if (lane == 0) s_red[warp][k] = r;
  }
  __syncthreads();
  if (threadIdx.x < NV) {
    double r = 0.0;
#pragma unroll
    for (int w = 0; w < kLinBlock / 32; w++) r += s_red[w][threadIdx.x];
    partial[(size_t)blockIdx.x * NV + threadIdx.x] = r;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(counter, 1u);
    s_last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    if (threadIdx.x < NV) {
      double r = 0.0;
      for (unsigned int b = 0; b < gridDim.x; b++) r += partial[(size_t)b * NV + threadIdx.x];
      s_tot[threadIdx.x] = r;
    }
    __syncthreads();
    if (comm.active()) {
      // multi-GPU: the last block exchanges this rank's sums with the peers through their segments (comm.cuh) and adds
      // the world's slots in rank order — the result the host reads is already the global one, bit-identical on all ranks
      comm_lm_publish(comm, xseq, s_tot, NV);
      comm_lm_collect(comm, xseq, s_tot, NV);  // a lost peer leaves the local sums in place after the poll budget
    }
    if (threadIdx.x < NV) {
      out[threadIdx.x] = s_tot[threadIdx.x];
      if (host_out) host_out[threadIdx.x] = s_tot[threadIdx.x];
    }
    if (host_out) {
      __threadfence_system();
      __syncthreads();  // s_last is block-uniform
    }
    if (threadIdx.x == 0) {
      *counter = 0u;  // ready for the next launch
      if (host_seq) publish_seq(host_seq, seq);
    }
  }
}

}  // namespace gsicp
