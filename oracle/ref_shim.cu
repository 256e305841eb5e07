// ref_shim.cu — C entry points around the REFERENCE's own CUDA code, compiled from the sources where
// they lie under /root/reference (never copied): oracle/Makefile builds this file together with
//   submodules/diff-gaussian-rasterization/cuda_rasterizer/{forward,backward,rasterizer_impl}.cu
//   submodules/simple-knn/simple_knn.cu
// into oracle/_ref/libref_cuda.so.  TEST INFRASTRUCTURE: used by tests/ (GPU parity, golden-vector
// generation) and by bench.py's per-kernel "reference CUDA on the same GPU" comparison only.
//
// Everything below is our own glue: it calls the reference's public C++ interface
// (cuda_rasterizer/rasterizer.h:22-88, simple_knn.h:15-19) with device pointers supplied by the caller.
#include <cuda_runtime.h>
#include <cstdint>
#include <functional>
#include <vector>

#include "cuda_rasterizer/rasterizer.h"
#include "cuda_rasterizer/rasterizer_impl.h"
#include "simple_knn.h"

namespace {
struct DevBuf {
  char* p = nullptr;
  size_t n = 0;
  char* resize(size_t bytes) {
    if (p) cudaFree(p);
    n = bytes;
    cudaMalloc(&p, bytes ? bytes : 1);
    return p;
  }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};
struct RefState {
  DevBuf geom, binning, img;
  int P = 0, R = 0, W = 0, H = 0;
};
}  // namespace

extern "C" {

void* ref_raster_forward(int P, int D, int M, const float* bg, int W, int H, const float* means3D, const float* shs,
                         const float* colors, const float* opac, const float* scales, float scale_mod,
                         const float* rots, const float* cov_pre, const float* view, const float* proj,
                         const float* campos, float tanx, float tany, int prefiltered, float* out_depth,
                         float* out_color, int* radii, bool* is_used, int* num_rendered) {
  RefState* st = new RefState();
  st->P = P; st->W = W; st->H = H;
  std::function<char*(size_t)> g = [st](size_t n) { return st->geom.resize(n); };
  std::function<char*(size_t)> b = [st](size_t n) { return st->binning.resize(n); };
  std::function<char*(size_t)> i = [st](size_t n) { return st->img.resize(n); };
  st->R = CudaRasterizer::Rasterizer::forward(g, b, i, P, D, M, bg, W, H, means3D, shs, colors, opac, scales, scale_mod,
                                              rots, cov_pre, view, proj, campos, tanx, tany, prefiltered != 0, out_depth,
                                              out_color, radii, is_used, false);
  cudaDeviceSynchronize();
  if (num_rendered) *num_rendered = st->R;
  return st;
}

int ref_raster_backward(void* handle, int D, int M, const float* bg, const float* means3D, const float* shs,
                        const float* colors, const float* scales, float scale_mod, const float* rots,
                        const float* cov_pre, const float* view, const float* proj, const float* campos, float tanx,
                        float tany, const int* radii, const float* dL_dpix_depth, const float* dL_dpix,
                        float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_ddepths, float* dL_dcolors,
                        float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot) {
  RefState* st = (RefState*)handle;
  CudaRasterizer::Rasterizer::backward(st->P, D, M, st->R, bg, st->W, st->H, means3D, shs, colors, scales, scale_mod,
                                       rots, cov_pre, view, proj, campos, tanx, tany, radii, st->geom.p, st->binning.p,
                                       st->img.p, dL_dpix_depth, dL_dpix, dL_dmean2D, dL_dconic, dL_dopacity,
                                       dL_ddepths, dL_dcolors, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, false);
  return (int)cudaDeviceSynchronize();
}

// sorted tile-instance list and per-tile ranges, read through the reference's own state layout
int ref_raster_export(void* handle, uint32_t* d_point_list, uint32_t* d_ranges) {
  RefState* st = (RefState*)handle;
  char* bp = st->binning.p;
  CudaRasterizer::BinningState bin = CudaRasterizer::BinningState::fromChunk(bp, st->R);
  char* ip = st->img.p;
  CudaRasterizer::ImageState img = CudaRasterizer::ImageState::fromChunk(ip, (size_t)st->W * st->H);
  if (st->R > 0) cudaMemcpy(d_point_list, bin.point_list, sizeof(uint32_t) * st->R, cudaMemcpyDeviceToDevice);
  const int tiles = ((st->W + 15) / 16) * ((st->H + 15) / 16);
  cudaMemcpy(d_ranges, img.ranges, sizeof(uint2) * tiles, cudaMemcpyDeviceToDevice);
  return (int)cudaDeviceSynchronize();
}

void ref_raster_free(void* handle) { delete (RefState*)handle; }

// timing helper: runs the reference forward `iters` times on fixed inputs (state discarded)
int ref_mark_visible(int P, float* means3D, float* view, float* proj, bool* present) {
  CudaRasterizer::Rasterizer::markVisible(P, means3D, view, proj, present);
  return (int)cudaDeviceSynchronize();
}

int ref_dist2(int P, float* points, float* out) {
  SimpleKNN::knn(P, (float3*)points, out);
  return (int)cudaDeviceSynchronize();
}

}  // extern "C"
