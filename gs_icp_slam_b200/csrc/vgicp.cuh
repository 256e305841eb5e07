// vgicp.cuh — voxelized GICP (pygicp.FastVGICP) on the GPU: the target's Gaussian voxel map and the voxel-correspondence
// normal equations, launched by the host-driven LM loop of gicp.cu.  Kernels in vgicp.cu (compiled with -fmad=false).
#pragma once
#include "host_common.h"
#include "gicp_reduce.cuh"

namespace gsicp {

constexpr int kVoxelBits = 21;  // bits per axis of a packed voxel key (coordinate minus the map's smallest coordinate)

// GaussianVoxelMap in ADDITIVE mode (FG/include/fast_gicp/gicp/fast_vgicp_voxel.hpp:105-186): per voxel the mean of its
// points, the mean of their covariances and the point count.  Voxels are stored in ascending packed-key order.
struct VoxelMap {
  int n = 0;                    // voxels; 0 = no map
  double res = 0.0;             // resolution the map was built with
  int lo[3] = {0, 0, 0};        // smallest voxel coordinate per axis
  int dim[3] = {0, 0, 0};       // extent in voxels per axis (< 2^kVoxelBits)
  Scratch coord;                // int [3 * points]; then the bounding box / status words
  Scratch bbox;                 // uint [7]: order-preserving min xyz, max xyz, out-of-range flag
  Scratch keys_in, idx_in, keys, idx;  // packed key and point index, before and after the stable sort
  Scratch ukeys, count, start, nvox;   // run-length encoding: voxel key, points, first sorted slot; voxel count
  Scratch mean, cov;            // double [3 * n], [6 * n] (upper triangle)
  Scratch cub_tmp;
};

struct VoxelView {  // by value into the kernels
  int n;
  double res;
  int lo[3], dim[3];
  const unsigned long long* keys;
  const int* count;
  const double* mean;
  const double* cov;
};

struct VgicpArgs {
  VoxelView vox;
  int n_src, n_offsets;           // n_offsets: 1, 7 or 27 (DIRECT1 / DIRECT7 / DIRECT27)
  const float* src_xyz;
  const double* src_cov;
  double* partial;
  double* out;
  unsigned int* counter;
  double* host_out;               // mapped pinned or null (see block_reduce_finalize)
  volatile unsigned long long* host_seq;
  unsigned long long seq;
};

// Build the map of n points (fp32 xyz, 6-double covariances) at resolution res.  GSICP_EINVAL when a coordinate is
// not finite, does not fit an int, or the extent needs more than kVoxelBits bits on an axis.  Synchronises the stream.
int voxelmap_build(VoxelMap& m, const float* xyz, const double* cov, int n, double res, cudaStream_t stream);
void voxelmap_free(VoxelMap& m);
VoxelView voxelmap_view(const VoxelMap& m);
// means [n][4] (w = 1) and covariances [n][16] (mirrored triangle, row and column 3 zero), in key order.
int voxelmap_export(const VoxelMap& m, double* means, double* covs, cudaStream_t stream);

// fast_vgicp_impl.hpp:73-180 at pose T: H (21), b (6) and the error (1) through block_reduce_finalize<kRed>.
int vgicp_launch_linearize(const VgicpArgs& a, const PoseD& T, cudaStream_t stream);
// fast_vgicp_impl.hpp:183-204: the error at Ti of the voxel pairs and Mahalanobis matrices of the linearisation pose T0.
int vgicp_launch_error(const VgicpArgs& a, const PoseD& T0, const PoseD& Ti, cudaStream_t stream);

}  // namespace gsicp
