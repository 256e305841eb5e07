// knn_dist2.cu — distCUDA2: mean squared distance to the 3 nearest other points.
//
// Replaces SimpleKNN::knn (submodules/simple-knn/simple_knn.cu:185-221: bbox reduce with two D2H copies ->
// 30-bit Morton codes -> radix sort -> 1024-point boxes -> per-point scan of every box that cannot be
// rejected).  Here: one uniform-grid build (grid.cuh, no host sync) and one exact 3-NN query per point.
// The result is the mathematically defined quantity the reference computes (self excluded by index,
// coincident points count with distance 0), so parity is to fp32 rounding of the distances.
#include "grid.cuh"

namespace gsicp {

// one warp per point: exact 3-NN excluding the point itself
__global__ void __launch_bounds__(128)
dist2_kernel(GridView g, const float* __restrict__ xyz, float* __restrict__ out) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= g.n) return;  // warp-uniform
  float d2;
  uint32_t id;
  grid_knn_warp(g, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], 3, (uint32_t)i, d2, id);
  const float a = __shfl_sync(0xffffffffu, d2, 0), b = __shfl_sync(0xffffffffu, d2, 1), c = __shfl_sync(0xffffffffu, d2, 2);
  if ((threadIdx.x & 31) == 0) out[i] = (a + b + c) / 3.0f;
}

static DeviceGrid g_dist2_grid;
static std::mutex g_dist2_mu;

// Geometry of the grid of the last distCUDA2 call (test hook gsicp_test_grid_meta); GSICP_ESTATE before the first call.
int dist2_grid_meta(GridMeta* out) {
  std::lock_guard<std::mutex> lock(g_dist2_mu);
  if (g_dist2_grid.n <= 0 || !g_dist2_grid.meta_buf.ptr) {
    set_error("gsicp_test_grid_meta: distCUDA2 has not built a grid yet");
    return GSICP_ESTATE;
  }
  GSICP_CUDA(cudaDeviceSynchronize());
  GSICP_CUDA(cudaMemcpy(out, g_dist2_grid.meta_buf.ptr, sizeof(GridMeta), cudaMemcpyDeviceToHost));
  return GSICP_OK;
}

}  // namespace gsicp

using namespace gsicp;

extern "C" int gsicp_dist2(int P, const float* d_points, float* d_out, void* stream_v) {
  if (P < 0 || (P > 0 && (!d_points || !d_out))) {
    set_error("gsicp_dist2: bad arguments");
    return GSICP_EINVAL;
  }
  if (P == 0) return GSICP_OK;
  cudaStream_t stream = (cudaStream_t)stream_v;
  std::lock_guard<std::mutex> lock(g_dist2_mu);
  ProfScope ps(kProfDist2, stream);
  if (int e = g_dist2_grid.build(d_points, P, stream)) return e;
  GSICP_LAUNCH(dist2_kernel, (int)(((size_t)P * 32 + 127) / 128), 128, 0, stream, g_dist2_grid.view(), d_points, d_out);
  GSICP_CUDA(cudaGetLastError());
  return GSICP_OK;
}
