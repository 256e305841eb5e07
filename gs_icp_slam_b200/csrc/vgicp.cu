// vgicp.cu — voxelized GICP on the GPU behind the pygicp.FastVGICP interface.
//
// Replaces fast_gicp::FastVGICP<PointXYZ,PointXYZ> (CPU, OpenMP, std::unordered_map of voxels):
//   fvi = FG/include/fast_gicp/gicp/impl/fast_vgicp_impl.hpp ; fvv = FG/include/fast_gicp/gicp/fast_vgicp_voxel.hpp
//
//   voxel map            fvv:129-160  ADDITIVE GaussianVoxelMap of the target: voxel coordinate floor(x / res - 0.5) per
//                        axis; the coordinates are packed into 64-bit keys relative to the smallest one (21 bits per axis),
//                        stable-sorted with their point index, run-length encoded, and one thread per voxel sums its points
//                        IN INDEX ORDER in fp64 — the reference's append() sequence, so the voxel means are bit-identical
//   vgicp_linearize      fvi:73-180   one thread per source point: fp64 transform, voxel coordinate, DIRECT1/7/27 offsets
//                        looked up by binary search in the sorted keys; per hit M = (C_B + R C_A R^T)^-1, w = sqrt(n_voxel),
//                        w e^T M e, w J^T M J, w J^T M e with J = [skew(q) | -I] -> 28-double block reduction
//   vgicp_error          fvi:183-204  w e^T M e at a trial pose with the pairs and M of the linearisation pose: both are
//                        recomputed from that pose with the same arithmetic (identical values), so nothing is stored per pair
//
// max_correspondence_distance plays no part, as in the reference.  Compiled with -fmad=false (the voxel coordinate of a
// transformed point depends on every rounding).
#include <cmath>
#include <vector>
#include <cub/cub.cuh>
#include "vgicp.cuh"

namespace gsicp {

// fvv:10-44 neighbor_offsets: DIRECT1 is the first entry of DIRECT7
__constant__ int c_off7[7][3] = {{0, 0, 0}, {1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
__constant__ int c_off27[27][3] = {
    {-1, -1, -1}, {-1, -1, 0}, {-1, -1, 1}, {-1, 0, -1}, {-1, 0, 0}, {-1, 0, 1}, {-1, 1, -1}, {-1, 1, 0}, {-1, 1, 1},
    {0, -1, -1},  {0, -1, 0},  {0, -1, 1},  {0, 0, -1},  {0, 0, 0},  {0, 0, 1},  {0, 1, -1},  {0, 1, 0},  {0, 1, 1},
    {1, -1, -1},  {1, -1, 0},  {1, -1, 1},  {1, 0, -1},  {1, 0, 0},  {1, 0, 1},  {1, 1, -1},  {1, 1, 0},  {1, 1, 1}};

// ------------------------------------------------------------------------------------------------
// voxel map
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int ord_u32(int x) { return (unsigned int)x ^ 0x80000000u; }  // order-preserving
static int from_ord_u32(unsigned int u) { return (int)(u ^ 0x80000000u); }

// fvv:158-160 voxel_coord: (x / res - 0.5).floor().cast<int>(); bbox = {min xyz, max xyz} as ord_u32, bbox[6] = 1 when a
// coordinate is not finite or does not fit an int (the reference's cast is undefined there)
__global__ void voxel_coord_kernel(int n, const float* __restrict__ xyz, double res, int* __restrict__ coord,
                                   unsigned int* __restrict__ bbox) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
#pragma unroll
  for (int d = 0; d < 3; d++) {
    const double c = floor((double)xyz[3 * (size_t)i + d] / res - 0.5);
    int ci = 0;
    if (c >= -2147483648.0 && c <= 2147483647.0) {
      ci = (int)c;
    } else {
      bbox[6] = 1u;
    }
    coord[3 * (size_t)i + d] = ci;
    atomicMin(bbox + d, ord_u32(ci));
    atomicMax(bbox + 3 + d, ord_u32(ci));
  }
}

__global__ void voxel_key_kernel(int n, const int* __restrict__ coord, int lx, int ly, int lz,
                                 unsigned long long* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long kx = (unsigned int)(coord[3 * (size_t)i] - lx);
  const unsigned long long ky = (unsigned int)(coord[3 * (size_t)i + 1] - ly);
  const unsigned long long kz = (unsigned int)(coord[3 * (size_t)i + 2] - lz);
  keys[i] = kx | (ky << kVoxelBits) | (kz << (2 * kVoxelBits));
  idx[i] = i;
}

// One thread per voxel: AdditiveGaussianVoxel::append over its points in index order (the stable sort keeps it), then
// finalize() (fvv:112-121).  The mean's w sums to n and divides back to 1; it is not stored.
__global__ void voxel_stats_kernel(int nv, const int* __restrict__ count, const int* __restrict__ start,
                                   const int* __restrict__ idx, const float* __restrict__ xyz, const double* __restrict__ cov,
                                   double* __restrict__ mean, double* __restrict__ vcov) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  const int c = count[v], s = start[v];
  double m[3] = {0.0, 0.0, 0.0}, C[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int j = s; j < s + c; j++) {
    const int p = idx[j];
#pragma unroll
    for (int d = 0; d < 3; d++) m[d] += (double)xyz[3 * (size_t)p + d];
#pragma unroll
    for (int k = 0; k < 6; k++) C[k] += cov[6 * (size_t)p + k];
  }
  const double nd = (double)c;
#pragma unroll
  for (int d = 0; d < 3; d++) mean[3 * (size_t)v + d] = m[d] / nd;
#pragma unroll
  for (int k = 0; k < 6; k++) vcov[6 * (size_t)v + k] = C[k] / nd;
}

// ------------------------------------------------------------------------------------------------
// linearize / error
// ------------------------------------------------------------------------------------------------
// Isometry3d * Vector4d (w = 1) in the order Eigen evaluates it (Transform.h: a 3x4 lazy product; rows 0-1 form one SSE2
// packet, ((c0 x + c1 y) + c2 z) + c3, row 2 is a scalar tree reduction, (c0 x + c1 y) + (c2 z + c3)).  Checked against
// the reference build's compiler flags.
__device__ __forceinline__ void transform_f64(const PoseD& T, double ax, double ay, double az, double q[3]) {
  q[0] = ((T.R[0][0] * ax + T.R[0][1] * ay) + T.R[0][2] * az) + T.t[0];
  q[1] = ((T.R[1][0] * ax + T.R[1][1] * ay) + T.R[1][2] * az) + T.t[1];
  q[2] = (T.R[2][0] * ax + T.R[2][1] * ay) + (T.R[2][2] * az + T.t[2]);
}

// Voxel at floor()ed coordinate (cx, cy, cz), or -1: outside the map's box, or not in the sorted keys (binary search).
__device__ __forceinline__ int voxel_find(const VoxelView& v, double cx, double cy, double cz) {
  const double rx = cx - (double)v.lo[0], ry = cy - (double)v.lo[1], rz = cz - (double)v.lo[2];
  if (!(rx >= 0.0 && rx < (double)v.dim[0] && ry >= 0.0 && ry < (double)v.dim[1] && rz >= 0.0 && rz < (double)v.dim[2]))
    return -1;  // also NaN
  const unsigned long long key =
      (unsigned long long)rx | ((unsigned long long)ry << kVoxelBits) | ((unsigned long long)rz << (2 * kVoxelBits));
  int lo = 0, hi = v.n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(v.keys + mid) < key) lo = mid + 1;
    else hi = mid;
  }
  return (lo < v.n && __ldg(v.keys + lo) == key) ? lo : -1;
}

// M = (C_B + R C_A R^T)^-1 of one (source point, voxel) pair (fvi:110-114); RA = R C_A.  A singular sum contributes nothing.
__device__ __forceinline__ void pair_mahalanobis(const PoseD& T, const double RA[3][3], const double* __restrict__ cb,
                                                 double M[3][3]) {
  const double B[3][3] = {{cb[0], cb[1], cb[2]}, {cb[1], cb[3], cb[4]}, {cb[2], cb[4], cb[5]}};
  double RCR[3][3];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) RCR[r][c] = B[r][c] + ((RA[r][0] * T.R[c][0] + RA[r][1] * T.R[c][1]) + RA[r][2] * T.R[c][2]);
  if (!inverse3(RCR, M)) {
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int c = 0; c < 3; c++) M[r][c] = 0.0;
  }
}

// The voxel pairs of source point i at the linearisation pose T0 (fvi:83-94): calls f(voxel, M) for every hit, in offset
// order.  Shared by linearize and error, so both see the same pairs and bit-identical M.
template <typename F>
__device__ __forceinline__ void for_each_pair(const VgicpArgs& a, const PoseD& T0, int i, const double q0[3], F&& f) {
  const double* ca = a.src_cov + 6 * (size_t)i;
  const double A[3][3] = {{ca[0], ca[1], ca[2]}, {ca[1], ca[3], ca[4]}, {ca[2], ca[4], ca[5]}};
  double RA[3][3];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) RA[r][c] = (T0.R[r][0] * A[0][c] + T0.R[r][1] * A[1][c]) + T0.R[r][2] * A[2][c];
  const double res = a.vox.res;
  const double cx = floor(q0[0] / res - 0.5), cy = floor(q0[1] / res - 0.5), cz = floor(q0[2] / res - 0.5);
  for (int o = 0; o < a.n_offsets; o++) {
    const int* off = a.n_offsets == 27 ? c_off27[o] : c_off7[o];
    const int k = voxel_find(a.vox, cx + off[0], cy + off[1], cz + off[2]);
    if (k < 0) continue;
    double M[3][3];
    pair_mahalanobis(T0, RA, a.vox.cov + 6 * (size_t)k, M);
    f(k, M);
  }
}

__global__ void __launch_bounds__(kLinBlock, 1)
vgicp_linearize_kernel(PoseD T, VgicpArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v[kRed];
#pragma unroll
  for (int k = 0; k < kRed; k++) v[k] = 0.0;
  if (i < a.n_src) {
    double q[3];
    transform_f64(T, (double)a.src_xyz[3 * (size_t)i], (double)a.src_xyz[3 * (size_t)i + 1], (double)a.src_xyz[3 * (size_t)i + 2], q);
    // J = [S | -I], S = skew(q) (fvi:156-158)
    const double S[3][3] = {{0.0, -q[2], q[1]}, {q[2], 0.0, -q[0]}, {-q[1], q[0], 0.0}};
    for_each_pair(a, T, i, q, [&](int k, const double M[3][3]) {
      const double w = sqrt((double)__ldg(a.vox.count + k));
      const double* mb = a.vox.mean + 3 * (size_t)k;
      const double e[3] = {mb[0] - q[0], mb[1] - q[1], mb[2] - q[2]};
      double Me[3];
#pragma unroll
      for (int r = 0; r < 3; r++) Me[r] = (M[r][0] * e[0] + M[r][1] * e[1]) + M[r][2] * e[2];
      v[27] += w * ((e[0] * Me[0] + e[1] * Me[1]) + e[2] * Me[2]);
      double MS[3][3];
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) MS[r][c] = (M[r][0] * S[0][c] + M[r][1] * S[1][c]) + M[r][2] * S[2][c];
      double H[6][6];
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) {
          H[r][c] = (S[0][r] * MS[0][c] + S[1][r] * MS[1][c]) + S[2][r] * MS[2][c];      // S^T M S
          H[r][3 + c] = -((S[0][r] * M[0][c] + S[1][r] * M[1][c]) + S[2][r] * M[2][c]);  // -S^T M
          H[3 + r][3 + c] = M[r][c];
        }
      int o = 0;
#pragma unroll
      for (int r = 0; r < 6; r++)
#pragma unroll
        for (int c = r; c < 6; c++) v[o++] += w * H[r][c];
#pragma unroll
      for (int r = 0; r < 3; r++) {
        v[21 + r] += w * ((S[0][r] * Me[0] + S[1][r] * Me[1]) + S[2][r] * Me[2]);  // S^T M e
        v[24 + r] += w * -Me[r];
      }
    });
  }
  block_reduce_finalize<kRed>(v, a.partial, a.out, a.counter, a.host_out, a.host_seq, a.seq);
}

__global__ void __launch_bounds__(kLinBlock)
vgicp_error_kernel(PoseD T0, PoseD Ti, VgicpArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v[1] = {0.0};
  if (i < a.n_src) {
    const double ax = (double)a.src_xyz[3 * (size_t)i], ay = (double)a.src_xyz[3 * (size_t)i + 1], az = (double)a.src_xyz[3 * (size_t)i + 2];
    double q0[3], qi[3];
    transform_f64(T0, ax, ay, az, q0);
    transform_f64(Ti, ax, ay, az, qi);
    for_each_pair(a, T0, i, q0, [&](int k, const double M[3][3]) {
      const double w = sqrt((double)__ldg(a.vox.count + k));
      const double* mb = a.vox.mean + 3 * (size_t)k;
      const double e[3] = {mb[0] - qi[0], mb[1] - qi[1], mb[2] - qi[2]};
      double Me[3];
#pragma unroll
      for (int r = 0; r < 3; r++) Me[r] = (M[r][0] * e[0] + M[r][1] * e[1]) + M[r][2] * e[2];
      v[0] += w * ((e[0] * Me[0] + e[1] * Me[1]) + e[2] * Me[2]);
    });
  }
  block_reduce_finalize<1>(v, a.partial, a.out, a.counter, a.host_out, a.host_seq, a.seq);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int voxelmap_build(VoxelMap& m, const float* xyz, const double* cov, int n, double res, cudaStream_t stream) {
  m.n = 0;
  if (!(std::isfinite(res) && res > 0.0)) {
    set_error("voxel resolution must be finite and > 0 (got %g)", res);
    return GSICP_EINVAL;
  }
  if (n <= 0) return GSICP_OK;
  const size_t nn = (size_t)n;
  if (int e = m.coord.ensure(nn * 3 * sizeof(int))) return e;
  if (int e = m.bbox.ensure(8 * sizeof(unsigned int))) return e;
  if (int e = m.keys_in.ensure(nn * sizeof(unsigned long long))) return e;
  if (int e = m.keys.ensure(nn * sizeof(unsigned long long))) return e;
  if (int e = m.ukeys.ensure(nn * sizeof(unsigned long long))) return e;
  if (int e = m.idx_in.ensure(nn * sizeof(int))) return e;
  if (int e = m.idx.ensure(nn * sizeof(int))) return e;
  if (int e = m.count.ensure(nn * sizeof(int))) return e;
  if (int e = m.start.ensure(nn * sizeof(int))) return e;
  if (int e = m.nvox.ensure(sizeof(int))) return e;
  if (int e = m.mean.ensure(nn * 3 * sizeof(double))) return e;
  if (int e = m.cov.ensure(nn * 6 * sizeof(double))) return e;

  unsigned int* bbox = m.bbox.as<unsigned int>();
  GSICP_CUDA(cudaMemsetAsync(bbox, 0xff, 3 * sizeof(unsigned int), stream));
  GSICP_CUDA(cudaMemsetAsync(bbox + 3, 0, 4 * sizeof(unsigned int), stream));
  const int blocks = (n + 255) / 256;
  GSICP_LAUNCH(voxel_coord_kernel, blocks, 256, 0, stream, n, xyz, res, m.coord.as<int>(), bbox);
  unsigned int hb[7];
  GSICP_CUDA(cudaMemcpyAsync(hb, bbox, sizeof(hb), cudaMemcpyDeviceToHost, stream));
  GSICP_CUDA(cudaStreamSynchronize(stream));
  if (hb[6]) {
    set_error("voxel map: a target coordinate is not finite or its voxel index does not fit an int at resolution %g", res);
    return GSICP_EINVAL;
  }
  int lo[3], dim[3];
  for (int d = 0; d < 3; d++) {
    lo[d] = from_ord_u32(hb[d]);
    const long long ext = (long long)from_ord_u32(hb[3 + d]) - lo[d] + 1;
    if (ext > (1ll << kVoxelBits)) {
      set_error("voxel map: the target spans %lld voxels on axis %d at resolution %g (at most 2^%d)", ext, d, res, kVoxelBits);
      return GSICP_EINVAL;
    }
    dim[d] = (int)ext;
  }
  GSICP_LAUNCH(voxel_key_kernel, blocks, 256, 0, stream, n, m.coord.as<int>(), lo[0], lo[1], lo[2],
               m.keys_in.as<unsigned long long>(), m.idx_in.as<int>());

  size_t t_sort = 0, t_rle = 0, t_scan = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t_sort, m.keys_in.as<unsigned long long>(), m.keys.as<unsigned long long>(),
                                  m.idx_in.as<int>(), m.idx.as<int>(), n, 0, 3 * kVoxelBits, stream);
  cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, m.keys.as<unsigned long long>(), m.ukeys.as<unsigned long long>(),
                                     m.count.as<int>(), m.nvox.as<int>(), n, stream);
  cub::DeviceScan::ExclusiveSum(nullptr, t_scan, m.count.as<int>(), m.start.as<int>(), n, stream);
  if (int e = m.cub_tmp.ensure(std::max(t_sort, std::max(t_rle, t_scan)))) return e;
  size_t tmp = m.cub_tmp.cap;
  // LSD radix sort: stable, so every voxel's points stay in index order
  GSICP_CUDA(cub::DeviceRadixSort::SortPairs(m.cub_tmp.ptr, tmp, m.keys_in.as<unsigned long long>(), m.keys.as<unsigned long long>(),
                                             m.idx_in.as<int>(), m.idx.as<int>(), n, 0, 3 * kVoxelBits, stream));
  tmp = m.cub_tmp.cap;
  GSICP_CUDA(cub::DeviceRunLengthEncode::Encode(m.cub_tmp.ptr, tmp, m.keys.as<unsigned long long>(), m.ukeys.as<unsigned long long>(),
                                                m.count.as<int>(), m.nvox.as<int>(), n, stream));
  int nv = 0;
  GSICP_CUDA(cudaMemcpyAsync(&nv, m.nvox.ptr, sizeof(int), cudaMemcpyDeviceToHost, stream));
  GSICP_CUDA(cudaStreamSynchronize(stream));
  tmp = m.cub_tmp.cap;
  GSICP_CUDA(cub::DeviceScan::ExclusiveSum(m.cub_tmp.ptr, tmp, m.count.as<int>(), m.start.as<int>(), nv, stream));
  GSICP_LAUNCH(voxel_stats_kernel, (nv + 127) / 128, 128, 0, stream, nv, m.count.as<int>(), m.start.as<int>(), m.idx.as<int>(),
               xyz, cov, m.mean.as<double>(), m.cov.as<double>());
  GSICP_CUDA(cudaGetLastError());
  m.n = nv;
  m.res = res;
  for (int d = 0; d < 3; d++) {
    m.lo[d] = lo[d];
    m.dim[d] = dim[d];
  }
  return GSICP_OK;
}

void voxelmap_free(VoxelMap& m) {
  for (Scratch* s : {&m.coord, &m.bbox, &m.keys_in, &m.idx_in, &m.keys, &m.idx, &m.ukeys, &m.count, &m.start, &m.nvox, &m.mean,
                     &m.cov, &m.cub_tmp}) {
    if (s->ptr) cudaFree(s->ptr);
    s->ptr = nullptr;
    s->cap = 0;
  }
  m.n = 0;
}

VoxelView voxelmap_view(const VoxelMap& m) {
  VoxelView v;
  v.n = m.n;
  v.res = m.res;
  for (int d = 0; d < 3; d++) {
    v.lo[d] = m.lo[d];
    v.dim[d] = m.dim[d];
  }
  v.keys = m.ukeys.as<unsigned long long>();
  v.count = m.count.as<int>();
  v.mean = m.mean.as<double>();
  v.cov = m.cov.as<double>();
  return v;
}

int voxelmap_export(const VoxelMap& m, double* means, double* covs, cudaStream_t stream) {
  if (m.n == 0) return GSICP_OK;
  if (!means || !covs) return GSICP_EINVAL;
  std::vector<double> mu((size_t)m.n * 3), c((size_t)m.n * 6);
  GSICP_CUDA(cudaMemcpyAsync(mu.data(), m.mean.ptr, mu.size() * sizeof(double), cudaMemcpyDeviceToHost, stream));
  GSICP_CUDA(cudaMemcpyAsync(c.data(), m.cov.ptr, c.size() * sizeof(double), cudaMemcpyDeviceToHost, stream));
  GSICP_CUDA(cudaStreamSynchronize(stream));
  for (int v = 0; v < m.n; v++) {
    double* o = means + 4 * (size_t)v;
    o[0] = mu[3 * (size_t)v]; o[1] = mu[3 * (size_t)v + 1]; o[2] = mu[3 * (size_t)v + 2]; o[3] = 1.0;
    const double* s = &c[6 * (size_t)v];
    double* C = covs + 16 * (size_t)v;
    const double full[16] = {s[0], s[1], s[2], 0.0, s[1], s[3], s[4], 0.0, s[2], s[4], s[5], 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < 16; k++) C[k] = full[k];
  }
  return GSICP_OK;
}

int vgicp_launch_linearize(const VgicpArgs& a, const PoseD& T, cudaStream_t stream) {
  const int blocks = std::max(1, (a.n_src + kLinBlock - 1) / kLinBlock);
  GSICP_LAUNCH(vgicp_linearize_kernel, blocks, kLinBlock, 0, stream, T, a);
  GSICP_CUDA(cudaGetLastError());
  return GSICP_OK;
}

int vgicp_launch_error(const VgicpArgs& a, const PoseD& T0, const PoseD& Ti, cudaStream_t stream) {
  const int blocks = std::max(1, (a.n_src + kLinBlock - 1) / kLinBlock);
  GSICP_LAUNCH(vgicp_error_kernel, blocks, kLinBlock, 0, stream, T0, Ti, a);
  GSICP_CUDA(cudaGetLastError());
  return GSICP_OK;
}

}  // namespace gsicp
