// host_common.h — host-side helpers shared by every translation unit of libgsicp_b200.so (and the device half of the
// mailbox protocol).
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include "../../include/gsicp_b200.h"

namespace gsicp {

extern std::atomic<uint64_t> g_launches;
void set_error(const char* fmt, ...);

// Counts every kernel launch of ours; bench.py reports it as gpu_launches.  With GSICP_DEBUG_SYNC=1 in the environment every
// launch is followed by a stream synchronize and the first failing kernel is named on stderr (debugging aid only).
extern int g_debug_sync;
void debug_sync_report(const char* kernel, cudaStream_t stream);
#define GSICP_LAUNCH(kernel, grid, block, smem, stream, ...)          \
  do {                                                                \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);       \
    ::gsicp::g_launches.fetch_add(1, std::memory_order_relaxed);      \
    if (::gsicp::g_debug_sync) ::gsicp::debug_sync_report(#kernel, (stream)); \
  } while (0)

#define GSICP_CUDA(expr)                                                                  \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::gsicp::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return GSICP_ECUDA;                                                                 \
    }                                                                                     \
  } while (0)

// Optional per-kernel device timing (bench.py roofline leg): when enabled, the hot kernels are bracketed by
// CUDA events recorded on the launching stream; totals are resolved when read.  Off by default.
enum ProfKernel {
  kProfPreprocess = 0, kProfDepthSort, kProfEmit, kProfTileSort, kProfRenderFwd, kProfRenderBwd, kProfGaussBwd,
  kProfCovariance, kProfLinearize, kProfError, kProfGridBuild, kProfDist2, kProfLossFwd, kProfLossBwd, kProfExchange, kProfCount
};
extern bool g_prof_on;
void prof_begin(int k, cudaStream_t s);
void prof_end(int k, cudaStream_t s);
struct ProfScope {
  int k; cudaStream_t s;
  ProfScope(int kk, cudaStream_t ss) : k(kk), s(ss) { if (g_prof_on) prof_begin(k, s); }
  ~ProfScope() { if (g_prof_on) prof_end(k, s); }
};

// Multiprocessors of the current device: persistent and grid-stride kernels size their grids by it.
inline int device_sm_count() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 1;  // the launch that follows reports the device error
  return sms > 0 ? sms : 1;
}

// Grow-only device scratch buffer (library-internal workspace that backward does not need).
struct Scratch {
  void* ptr = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return GSICP_OK;
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    cudaError_t e = cudaMalloc(&ptr, want);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
      return GSICP_ECUDA;
    }
    cap = want;
    return GSICP_OK;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(ptr); }
};

// ---- mailbox: values a kernel publishes to the host without a blocking copy -------------------------------------------
// The kernel writes its payload into mapped pinned memory and then publish_seq() stores a sequence word; the host spins in
// wait_published() until the word holds the sequence number it expects and then reads the payload.  Each caller owns its
// payload layout and its sequence counter.

// n zeroed elements of mapped pinned host memory (h) and their device alias (d).  alloc() allocates on the first call
// only; free() releases the block.
template <typename T>
struct Mapped {
  T* h = nullptr;
  T* d = nullptr;
  cudaError_t alloc(size_t n) {
    if (h) return cudaSuccess;
    cudaError_t e = cudaHostAlloc((void**)&h, n * sizeof(T), cudaHostAllocMapped);
    if (e != cudaSuccess) {
      h = nullptr;
      return e;
    }
    std::memset((void*)h, 0, n * sizeof(T));
    e = cudaHostGetDevicePointer((void**)&d, h, 0);
    if (e != cudaSuccess) free();
    return e;
  }
  void free() {
    if (h) cudaFreeHost(h);
    h = d = nullptr;
  }
};

// Spin until *word == seq.  Every 2^20 spins the stream is queried, so that a failed kernel ("<what> failed: ...") or a
// stream that went idle without publishing ("<what> was not published") returns GSICP_ECUDA instead of hanging.
int wait_published(const volatile unsigned long long* word, unsigned long long seq, cudaStream_t stream, const char* what);

#ifdef __CUDACC__
// Device half: call after the payload stores.  The fence makes the payload visible to the host before the sequence word.
__device__ __forceinline__ void publish_seq(volatile unsigned long long* word, unsigned long long seq) {
  __threadfence_system();
  *word = seq;
}
#endif

}  // namespace gsicp
