// comm.cu — host side of the multi-GPU exchange layer (comm.cuh): segment allocation, CUDA IPC mapping of the peers'
// segments, stream-ordered barrier.  One process per GPU; the 64-byte IPC handles travel over whatever channel the
// application has (torch.distributed.all_gather_object in gs_icp_slam_b200/sharding.py).
#include <cstring>
#include "comm.cuh"
#include "host_common.h"

namespace gsicp {

// One warp: lane r signals rank r (release: everything enqueued before on this stream is visible), then waits for
// rank r's signal.  Sequence numbers are monotone, so a fast peer's later signal also satisfies the wait.
__global__ void comm_barrier_kernel(CommView c, unsigned long long seq, int* status) {
  const int r = threadIdx.x;
  if (r < c.world) {
    __threadfence_system();
    unsigned long long* f = reinterpret_cast<unsigned long long*>(c.seg[r] + kCommBarOff) + c.rank;
    st_release_sys(f, seq);
    const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(c.seg[c.rank] + kCommBarOff) + r;
    long long polls = 0;
    while (ld_acquire_sys(mine) < seq) {
      if (++polls > kCommPollBudget) {
        if (status) *status = 1;
        break;
      }
    }
    __threadfence_system();
  }
}

int comm_preload_kernels() {
  cudaFuncAttributes fa;
  GSICP_CUDA(cudaFuncGetAttributes(&fa, (const void*)comm_barrier_kernel));
  return GSICP_OK;
}

int comm_stream_barrier(gsicp_comm* c, cudaStream_t stream) {
  if (!c || !c->connected || c->world <= 1) return GSICP_OK;
  if (c->status.h && *(volatile int*)c->status.h) {
    set_error("exchange group (rank %d of %d): an earlier barrier ran out of its poll budget - a peer did not arrive; results since "
              "then are not valid", c->rank, c->world);
    return GSICP_ECUDA;
  }
  const unsigned long long seq = ++c->bar_seq;
  GSICP_LAUNCH(comm_barrier_kernel, 1, 32, 0, stream, c->view(), seq, c->status.d);
  GSICP_CUDA(cudaGetLastError());
  return GSICP_OK;
}

}  // namespace gsicp

using namespace gsicp;

extern "C" int gsicp_comm_alloc(size_t heap_bytes, gsicp_comm** out, void* handle64) {
  if (!out || !handle64) return GSICP_EINVAL;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
  gsicp_comm* c = new gsicp_comm();
  auto fail = [&](int code, const char* what, cudaError_t e) {
    set_error("gsicp_comm_alloc: %s failed: %s", what, cudaGetErrorString(e));
    c->status.free();
    if (c->local) cudaFree(c->local);
    delete c;
    return code;
  };
  cudaError_t e = cudaGetDevice(&c->device);
  if (e != cudaSuccess) return fail(GSICP_ECUDA, "cudaGetDevice", e);
  c->bytes = kCommHeapOff + ((heap_bytes + 255) & ~size_t(255));
  if ((e = cudaMalloc((void**)&c->local, c->bytes)) != cudaSuccess) return fail(GSICP_ENOMEM, "cudaMalloc", e);
  if ((e = cudaMemset(c->local, 0, c->bytes)) != cudaSuccess) return fail(GSICP_ECUDA, "cudaMemset", e);
  if ((e = c->status.alloc(16)) != cudaSuccess) return fail(GSICP_ENOMEM, "mapped status allocation", e);
  cudaIpcMemHandle_t h;
  if ((e = cudaIpcGetMemHandle(&h, c->local)) != cudaSuccess) return fail(GSICP_ECUDA, "cudaIpcGetMemHandle", e);
  std::memcpy(handle64, &h, 64);
  *out = c;
  return GSICP_OK;
}

extern "C" int gsicp_comm_connect(gsicp_comm* c, int world, int rank, const void* handles) {
  if (!c || !handles || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) {
    set_error("gsicp_comm_connect: bad arguments (world %d, rank %d, max %d ranks)", world, rank, kMaxRanks);
    return GSICP_EINVAL;
  }
  c->world = world;
  c->rank = rank;
  for (int r = 0; r < world; r++) {
    if (r == rank) {
      c->peer[r] = c->local;
      continue;
    }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, (const char*)handles + 64 * (size_t)r, 64);
    void* p = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      set_error("gsicp_comm_connect: cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
      return GSICP_ECUDA;
    }
    c->peer[r] = (char*)p;
  }
  c->connected = true;
  return GSICP_OK;
}

// Test hook: connect the ranks of a group that live in ONE process on ONE device (CUDA IPC cannot map a process's own
// allocation): the peers' segments are given as plain device pointers.  Lets a single-GPU box exercise the device-side
// exchange protocols (two "ranks" on two streams).
extern "C" int gsicp_comm_connect_local(gsicp_comm* c, int world, int rank, gsicp_comm* const* group) {
  if (!c || !group || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) return GSICP_EINVAL;
  c->world = world;
  c->rank = rank;
  for (int r = 0; r < world; r++) {
    if (!group[r] || !group[r]->local) return GSICP_EINVAL;
    c->peer[r] = group[r]->local;
  }
  c->local_only = true;
  c->connected = true;
  return GSICP_OK;
}

extern "C" void gsicp_comm_destroy(gsicp_comm* c) {
  if (!c) return;
  for (int r = 0; r < c->world; r++)
    if (!c->local_only && r != c->rank && c->peer[r]) cudaIpcCloseMemHandle(c->peer[r]);
  if (c->local) cudaFree(c->local);
  c->status.free();
  delete c;
}

extern "C" int gsicp_comm_world(const gsicp_comm* c) { return c ? c->world : 0; }
extern "C" int gsicp_comm_rank(const gsicp_comm* c) { return c ? c->rank : -1; }

extern "C" int gsicp_comm_barrier(gsicp_comm* c, void* stream) { return comm_stream_barrier(c, (cudaStream_t)stream); }
