// flag_count.cuh — compaction offsets of the rows a 0/1 functor keeps: excl[i] = flag(0) + ... + flag(i - 1), and the
// one-thread kernel that publishes the kept-row count excl[n - 1] + flag(n - 1) to the host (mailbox, host_common.h).
#pragma once
#include <cub/cub.cuh>
#include "host_common.h"

namespace gsicp {

// Exclusive sum of flag(0 .. n-1) into excl (grown to n elements of T); cub_tmp is CUB's temporary storage.
template <typename T, typename Flag>
int flag_scan(int n, Flag flag, Scratch& excl, Scratch& cub_tmp, cudaStream_t stream) {
  if (int e = excl.ensure((size_t)n * sizeof(T))) return e;
  cub::CountingInputIterator<int> counting(0);
  cub::TransformInputIterator<T, Flag, cub::CountingInputIterator<int>> flags(counting, flag);
  size_t tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, flags, excl.as<T>(), n, stream);
  if (int e = cub_tmp.ensure(tmp)) return e;
  tmp = cub_tmp.cap;
  GSICP_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp.ptr, tmp, flags, excl.as<T>(), n, stream));
  return GSICP_OK;
}

template <typename T, typename Flag>
__global__ void publish_flag_count_kernel(int n, const T* __restrict__ excl, Flag flag, unsigned long long* count,
                                          unsigned long long* seq_word, unsigned long long seq) {
  *count = (unsigned long long)(excl[n - 1] + flag(n - 1));
  publish_seq(seq_word, seq);
}

}  // namespace gsicp
