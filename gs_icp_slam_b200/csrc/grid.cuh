// grid.cuh — exact nearest-neighbour search on a uniform cell grid, built and queried on the device.
//
// Replaces the reference's CPU kd-tree (pcl::search::KdTree -> FLANN KDTreeSingleIndex, exact, results
// sorted ascending; call sites fast_gicp_impl.hpp:268,401,616,737) and simple-knn's Morton boxes
// (simple_knn.cu:147-183).  A pointer-chasing tree is the wrong structure for a GPU; a dense cell grid
// with ring expansion gives the same EXACT answer with coalesced cell scans:
//   build : bbox -> cell size (on device, no host sync) -> cell histogram -> exclusive scan -> scatter
//           points into cell order as float4 {x, y, z, bits(original index)}.
//   query : visit the cube of cells of Chebyshev radius r = 0,1,2,... around the query; stop when the
//           k-th best squared distance is below the squared distance to the nearest unsearched face;
//           beyond kMaxRing rings fall back to a linear scan (queries far outside the cloud).
// Determinism: candidates are ordered by (squared distance, original index), so results do not depend on
// the scatter order; distances are computed as ((dx*dx) + dy*dy) + dz*dz in fp32 with no fma contraction,
// bit-identical to oracle/gicp_oracle.cpp.
#pragma once
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <float.h>
#include <mutex>
#include <stdint.h>
#include "host_common.h"

namespace gsicp {

struct GridMeta {  // lives in device memory; written by grid_setup_kernel
  float ox, oy, oz;  // origin (bbox min)
  float cell, inv_cell;
  int nx, ny, nz;
  int ncells;
};

struct GridView {  // passed by value to query kernels
  const GridMeta* meta;
  const uint32_t* cell_start;  // [max_cells + 1]
  const float4* pts;           // [n] in cell order: x, y, z, original index bits
  int n;
};

constexpr int kMaxRing = 6;

__device__ __forceinline__ float dist2_nofma(float ax, float ay, float az, float bx, float by, float bz) {
  const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// ---- build kernels ----------------------------------------------------------------------------
__device__ __forceinline__ unsigned int f2ord(float f) {  // order-preserving float -> uint
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned int u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

static __global__ void grid_bbox_init_kernel(unsigned int* bb) {
  if (threadIdx.x < 3) bb[threadIdx.x] = 0xffffffffu;
  else if (threadIdx.x < 6) bb[threadIdx.x] = 0u;
}

static __global__ void grid_bbox_kernel(int n, const float* __restrict__ xyz, unsigned int* bb) {
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      const float v = xyz[3 * (size_t)i + d];
      if (v == v) {  // ignore NaN coordinates
        mn[d] = fminf(mn[d], v);
        mx[d] = fmaxf(mx[d], v);
      }
    }
  }
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      atomicMin(&bb[d], f2ord(mn[d]));
      atomicMax(&bb[3 + d], f2ord(mx[d]));
    }
  }
}

// choose the cell size so that the dense grid has at most max_cells cells
__device__ __forceinline__ GridMeta grid_choose(const float lo_in[3], const float hi_in[3], int n, int max_cells) {
  float lo[3], hi[3], ext[3];
  for (int d = 0; d < 3; d++) {
    lo[d] = lo_in[d];
    hi[d] = hi_in[d];
    if (!(hi[d] >= lo[d])) { lo[d] = 0.f; hi[d] = 0.f; }
    ext[d] = hi[d] - lo[d];
  }
  const float emax = fmaxf(ext[0], fmaxf(ext[1], ext[2]));
  const double vol = (double)fmaxf(ext[0], emax * 1e-3f) * fmaxf(ext[1], emax * 1e-3f) * fmaxf(ext[2], emax * 1e-3f);
  // aim at ~2 cells per point (surfaces fill few cells; ~5-10 points per occupied cell)
  const double target = fmin((double)max_cells, fmax(64.0, 2.0 * (double)n));
  float cell = (float)cbrt(vol / target);
  if (!(cell > 0.f)) cell = 1.f;
  int nx = 1, ny = 1, nz = 1;
  for (int it = 0; it < 64; it++) {
    nx = (int)fminf(ext[0] / cell, 2.0e6f) + 1;
    ny = (int)fminf(ext[1] / cell, 2.0e6f) + 1;
    nz = (int)fminf(ext[2] / cell, 2.0e6f) + 1;
    if ((double)nx * ny * nz <= (double)max_cells) break;
    cell *= 1.25f;
  }
  GridMeta m;
  m.ox = lo[0]; m.oy = lo[1]; m.oz = lo[2];
  m.cell = cell;
  m.inv_cell = 1.0f / cell;
  m.nx = nx; m.ny = ny; m.nz = nz;
  m.ncells = nx * ny * nz;
  return m;
}

static __global__ void grid_setup_kernel(const unsigned int* bb, int n, int max_cells, GridMeta* meta) {
  float lo[3], hi[3];
  for (int d = 0; d < 3; d++) {
    lo[d] = ord2f(bb[d]);
    hi[d] = ord2f(bb[3 + d]);
  }
  *meta = grid_choose(lo, hi, n, max_cells);
}

// Coordinate of the lower face of cell k along one axis: o + k * cell, rounded twice whatever the translation unit's fma
// contraction setting, so that binning (grid_cell_of) and the stopping bound (ring_bound) agree on where every face is.
__device__ __forceinline__ float grid_face(float o, int k, float cell) { return __fadd_rn(o, __fmul_rn((float)k, cell)); }

// Cell of x along one axis.  The floor of (x - o) * inv_cell can land one cell off near a face (its two roundings differ
// from grid_face's, by up to ~1e-3 cell at cell index ~4000 when the box straddles 0); it is corrected against grid_face,
// so every binned point satisfies grid_face(i) <= x < grid_face(i + 1) except beyond the outer faces of the grid.
__device__ __forceinline__ int grid_axis_cell(float x, float o, float inv_cell, float cell, int n) {
  int c = (int)floorf(__fmul_rn(__fsub_rn(x, o), inv_cell));
  c = min(max(c, 0), n - 1);  // NaN/inf -> clamp (the int conversion of NaN is 0 on the device)
  if (x < grid_face(o, c, cell)) c = max(c - 1, 0);
  else if (x >= grid_face(o, c + 1, cell)) c = min(c + 1, n - 1);
  return c;
}

__device__ __forceinline__ int3 grid_cell_of(const GridMeta& m, float x, float y, float z) {
  return make_int3(grid_axis_cell(x, m.ox, m.inv_cell, m.cell, m.nx), grid_axis_cell(y, m.oy, m.inv_cell, m.cell, m.ny),
                   grid_axis_cell(z, m.oz, m.inv_cell, m.cell, m.nz));
}

static __global__ void grid_count_kernel(int n, const float* __restrict__ xyz, const GridMeta* __restrict__ meta,
                                  uint32_t* __restrict__ counts, uint32_t* __restrict__ cell_of_pt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const GridMeta m = *meta;
  const int3 c = grid_cell_of(m, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]);
  const uint32_t id = (uint32_t)((c.z * m.ny + c.y) * m.nx + c.x);
  cell_of_pt[i] = id;
  atomicAdd(&counts[id], 1u);
}

static __global__ void grid_scatter_kernel(int n, const float* __restrict__ xyz, const uint32_t* __restrict__ cell_of_pt,
                                    uint32_t* __restrict__ cursor, float4* __restrict__ pts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t slot = atomicAdd(&cursor[cell_of_pt[i]], 1u);
  pts[slot] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], __uint_as_float((uint32_t)i));
}

// Whole grid build in ONE CTA for small clouds (the tracker's 12k-point source cloud is rebuilt every frame): bbox,
// cell size, histogram, exclusive scan and scatter are phases of a single launch separated by block barriers instead of
// nine dependent launches (whose launch gaps, not their work, dominated).
constexpr int kSmallGridThreads = 1024;
constexpr int kSmallGridMaxPoints = 65536;

static __global__ void __launch_bounds__(kSmallGridThreads)
grid_build_small_kernel(int n, const float* __restrict__ xyz, int max_cells, GridMeta* __restrict__ meta_out,
                        uint32_t* __restrict__ cell_start, uint32_t* __restrict__ cursor, uint32_t* __restrict__ cell_of_pt,
                        float4* __restrict__ pts) {
  __shared__ float s_lo[3][32], s_hi[3][32];
  __shared__ GridMeta s_meta;
  __shared__ uint32_t s_part[kSmallGridThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // phase 1: bounding box
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int i = tid; i < n; i += kSmallGridThreads) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      const float v = xyz[3 * (size_t)i + d];
      if (v == v) {
        mn[d] = fminf(mn[d], v);
        mx[d] = fmaxf(mx[d], v);
      }
    }
  }
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
    if (lane == 0) {
      s_lo[d][warp] = mn[d];
      s_hi[d][warp] = mx[d];
    }
  }
  __syncthreads();
  if (tid == 0) {
    float lo[3], hi[3];
    for (int d = 0; d < 3; d++) {
      lo[d] = FLT_MAX;
      hi[d] = -FLT_MAX;
      for (int w = 0; w < kSmallGridThreads / 32; w++) {
        lo[d] = fminf(lo[d], s_lo[d][w]);
        hi[d] = fmaxf(hi[d], s_hi[d][w]);
      }
    }
    s_meta = grid_choose(lo, hi, n, max_cells);
    *meta_out = s_meta;
  }
  __syncthreads();
  const GridMeta m = s_meta;
  // phase 2: histogram of points per cell (cell_start doubles as the count array)
  for (int c = tid; c <= m.ncells; c += kSmallGridThreads) cell_start[c] = 0u;
  __syncthreads();
  for (int i = tid; i < n; i += kSmallGridThreads) {
    const int3 c = grid_cell_of(m, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]);
    const uint32_t id = (uint32_t)((c.z * m.ny + c.y) * m.nx + c.x);
    cell_of_pt[i] = id;
    atomicAdd(&cell_start[id], 1u);
  }
  __syncthreads();
  // phase 3: exclusive scan over the cells: each thread owns a contiguous chunk
  const int per = (m.ncells + kSmallGridThreads) / kSmallGridThreads;  // covers indices 0..ncells
  const int c0 = tid * per, c1 = min(c0 + per, m.ncells + 1);
  uint32_t local = 0;
  for (int c = c0; c < c1; c++) local += cell_start[c];
  uint32_t incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_part[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t v = s_part[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    s_part[lane] = v;  // inclusive over warps
  }
  __syncthreads();
  uint32_t run = (incl - local) + (warp > 0 ? s_part[warp - 1] : 0u);
  for (int c = c0; c < c1; c++) {
    const uint32_t cnt = cell_start[c];
    cell_start[c] = run;
    cursor[c] = run;
    run += cnt;
  }
  __syncthreads();
  // phase 4: scatter into cell order
  for (int i = tid; i < n; i += kSmallGridThreads) {
    const uint32_t slot = atomicAdd(&cursor[cell_of_pt[i]], 1u);
    pts[slot] = make_float4(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], __uint_as_float((uint32_t)i));
  }
}

// Same single-CTA build with the cell table in SHARED memory (clouds whose table fits: <= ~25k points, i.e. the
// tracker's per-frame source cloud): the histogram and the scatter cursor become shared-memory integer atomics and the scan
// never leaves the SM; global memory sees one read of xyz per phase (L1/L2 hits after the first) and one write of
// cell_start and pts.
constexpr int kSmemGridMaxCells = 50 * 1024;  // (cells + 1) * 4 B <= 200 KB of dynamic shared memory

static __global__ void __launch_bounds__(kSmallGridThreads)
grid_build_smem_kernel(int n, const float* __restrict__ xyz, int max_cells, GridMeta* __restrict__ meta_out,
                       uint32_t* __restrict__ cell_start, float4* __restrict__ pts) {
  extern __shared__ uint32_t s_cell[];  // [ncells + 1]: counts -> exclusive starts -> scatter cursors
  __shared__ float s_lo[3][32], s_hi[3][32];
  __shared__ GridMeta s_meta;
  __shared__ uint32_t s_part[kSmallGridThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int i = tid; i < n; i += kSmallGridThreads) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      const float v = xyz[3 * (size_t)i + d];
      if (v == v) {
        mn[d] = fminf(mn[d], v);
        mx[d] = fmaxf(mx[d], v);
      }
    }
  }
#pragma unroll
  for (int d = 0; d < 3; d++) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
    if (lane == 0) {
      s_lo[d][warp] = mn[d];
      s_hi[d][warp] = mx[d];
    }
  }
  for (int c = tid; c <= max_cells; c += kSmallGridThreads) s_cell[c] = 0u;
  __syncthreads();
  if (warp == 0) {
    float lo[3], hi[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
      lo[d] = s_lo[d][lane];
      hi[d] = s_hi[d][lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
        hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
      }
    }
    if (lane == 0) {
      s_meta = grid_choose(lo, hi, n, max_cells);
      *meta_out = s_meta;
    }
  }
  __syncthreads();
  const GridMeta m = s_meta;
  for (int i = tid; i < n; i += kSmallGridThreads) {
    const int3 c = grid_cell_of(m, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]);
    atomicAdd(&s_cell[(c.z * m.ny + c.y) * m.nx + c.x], 1u);
  }
  __syncthreads();
  const int per = (m.ncells + kSmallGridThreads) / kSmallGridThreads;  // covers indices 0..ncells
  const int c0 = min(tid * per, m.ncells + 1), c1 = min(c0 + per, m.ncells + 1);
  uint32_t local = 0;
  for (int c = c0; c < c1; c++) local += s_cell[c];
  uint32_t incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_part[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t v = s_part[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    s_part[lane] = v;
  }
  __syncthreads();
  uint32_t run = (incl - local) + (warp > 0 ? s_part[warp - 1] : 0u);
  for (int c = c0; c < c1; c++) {
    const uint32_t cnt = s_cell[c];
    s_cell[c] = run;
    run += cnt;
  }
  __syncthreads();
  for (int c = tid; c <= m.ncells; c += kSmallGridThreads) cell_start[c] = s_cell[c];
  __syncthreads();
  for (int i = tid; i < n; i += kSmallGridThreads) {
    const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
    const int3 c = grid_cell_of(m, x, y, z);
    const uint32_t slot = atomicAdd(&s_cell[(c.z * m.ny + c.y) * m.nx + c.x], 1u);
    pts[slot] = make_float4(x, y, z, __uint_as_float((uint32_t)i));
  }
}

// ---- device-side storage ----------------------------------------------------------------------
struct DeviceGrid {
  Scratch meta_buf, bbox_buf, cell_start, cursor, cell_of_pt, pts, cub_tmp;
  int n = 0, max_cells = 0;

  GridView view() const {
    GridView v;
    v.meta = meta_buf.as<GridMeta>();
    v.cell_start = cell_start.as<uint32_t>();
    v.pts = pts.as<float4>();
    v.n = n;
    return v;
  }

  // d_xyz: device (n,3) fp32.  All work is stream-ordered; no host synchronisation.
  int build(const float* d_xyz, int n_points, cudaStream_t stream) {
    n = n_points;
    if (n <= 0) return GSICP_OK;
    long long want = 2LL * n;
    if (want < 4096) want = 4096;
    if (want > (1LL << 24)) want = (1LL << 24);
    max_cells = (int)want;
    int e;
    if ((e = meta_buf.ensure(sizeof(GridMeta)))) return e;
    if ((e = bbox_buf.ensure(6 * sizeof(unsigned int)))) return e;
    if ((e = cell_start.ensure(((size_t)max_cells + 1) * 4))) return e;
    if ((e = cursor.ensure(((size_t)max_cells + 1) * 4))) return e;
    if ((e = cell_of_pt.ensure((size_t)n * 4))) return e;
    if ((e = pts.ensure((size_t)n * sizeof(float4)))) return e;
    size_t tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp, cursor.as<uint32_t>(), cell_start.as<uint32_t>(), max_cells + 1, stream);
    if ((e = cub_tmp.ensure(tmp))) return e;

    if (max_cells <= kSmemGridMaxCells) {
      static bool attr_set = false;
      const int smem = (max_cells + 1) * 4;
      if (!attr_set) {
        GSICP_CUDA(cudaFuncSetAttribute(grid_build_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (kSmemGridMaxCells + 1) * 4));
        attr_set = true;
      }
      GSICP_LAUNCH(grid_build_smem_kernel, 1, kSmallGridThreads, smem, stream, n, d_xyz, max_cells, meta_buf.as<GridMeta>(),
                   cell_start.as<uint32_t>(), pts.as<float4>());
      GSICP_CUDA(cudaGetLastError());
      return GSICP_OK;
    }
    if (n <= kSmallGridMaxPoints) {
      GSICP_LAUNCH(grid_build_small_kernel, 1, kSmallGridThreads, 0, stream, n, d_xyz, max_cells, meta_buf.as<GridMeta>(),
                   cell_start.as<uint32_t>(), cursor.as<uint32_t>(), cell_of_pt.as<uint32_t>(), pts.as<float4>());
      GSICP_CUDA(cudaGetLastError());
      return GSICP_OK;
    }
    GSICP_LAUNCH(grid_bbox_init_kernel, 1, 32, 0, stream, bbox_buf.as<unsigned int>());
    int blocks = (n + 255) / 256;
    if (blocks > 592) blocks = 592;
    GSICP_LAUNCH(grid_bbox_kernel, blocks, 256, 0, stream, n, d_xyz, bbox_buf.as<unsigned int>());
    GSICP_LAUNCH(grid_setup_kernel, 1, 1, 0, stream, bbox_buf.as<unsigned int>(), n, max_cells, meta_buf.as<GridMeta>());
    GSICP_CUDA(cudaMemsetAsync(cursor.ptr, 0, ((size_t)max_cells + 1) * 4, stream));
    GSICP_LAUNCH(grid_count_kernel, (n + 255) / 256, 256, 0, stream, n, d_xyz, meta_buf.as<GridMeta>(),
                 cursor.as<uint32_t>(), cell_of_pt.as<uint32_t>());
    tmp = cub_tmp.cap;
    GSICP_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp.ptr, tmp, cursor.as<uint32_t>(), cell_start.as<uint32_t>(),
                                             max_cells + 1, stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    GSICP_CUDA(cudaMemcpyAsync(cursor.ptr, cell_start.ptr, ((size_t)max_cells + 1) * 4, cudaMemcpyDeviceToDevice, stream));
    GSICP_LAUNCH(grid_scatter_kernel, (n + 255) / 256, 256, 0, stream, n, d_xyz, cell_of_pt.as<uint32_t>(),
                 cursor.as<uint32_t>(), pts.as<float4>());
    GSICP_CUDA(cudaGetLastError());
    return GSICP_OK;
  }
};

// ---- query ------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// Warp-cooperative exact search: ONE WARP PER QUERY (all 32 lanes call with the same query).
//
// Ring r of cells around the query cell consists of (2r+1)^2 x-rows.  Consecutive x cells own consecutive point
// ranges in `pts`, so a row on the shell of the ring is one contiguous range and an interior row contributes its two
// end cells: at most 2 "slots" per row.  The lanes compute the slots' [begin,end) in parallel, a warp scan flattens
// them, and the candidates are then read 32 at a time (coalesced float4 loads) regardless of how they are spread
// over cells.  The ring loop stops when `want` candidates are closer than the nearest unsearched cell face — an exact
// criterion; beyond kMaxRing rings (queries far outside the cloud) the warp scans the whole cloud linearly.
// ------------------------------------------------------------------------------------------------
struct RingCursor {  // warp-uniform description of the flattened candidate list of one group of 32 slots
  uint32_t b, excl, total;  // per lane: slot begin and exclusive prefix of the slot lengths; total is uniform
};

__device__ __forceinline__ RingCursor ring_slots(const GridView& g, const GridMeta& m, int3 c0, int r, int slot0, int lane) {
  const int side = 2 * r + 1;
  const int s = slot0 + lane;
  uint32_t b = 0, e = 0;
  if (s < 2 * side * side) {
    const int row = s >> 1, half = s & 1;
    const int dz = row / side - r, dy = row % side - r;
    const int z = c0.z + dz, y = c0.y + dy;
    if (z >= 0 && z < m.nz && y >= 0 && y < m.ny) {
      const int base = (z * m.ny + y) * m.nx;
      if (abs(dz) == r || abs(dy) == r) {
        if (half == 0) {
          b = g.cell_start[base + max(c0.x - r, 0)];
          e = g.cell_start[base + min(c0.x + r, m.nx - 1) + 1];
        }
      } else {
        const int x = half == 0 ? c0.x - r : c0.x + r;
        if (x >= 0 && x < m.nx) {
          b = g.cell_start[base + x];
          e = g.cell_start[base + x + 1];
        }
      }
    }
  }
  const uint32_t len = e - b;
  uint32_t incl = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  RingCursor c;
  c.b = b;
  c.excl = incl - len;
  c.total = __shfl_sync(0xffffffffu, incl, 31);
  return c;
}

// index into g.pts of flattened element t (t < total), for every lane independently
__device__ __forceinline__ uint32_t ring_element(const RingCursor& c, uint32_t t) {
  int lo = 0;  // largest slot k with excl[k] <= t
#pragma unroll
  for (int step = 16; step >= 1; step >>= 1) {
    const int probe = lo + step;
    const uint32_t v = __shfl_sync(0xffffffffu, c.excl, probe & 31);
    if (probe < 32 && v <= t) lo = probe;
  }
  const uint32_t sb = __shfl_sync(0xffffffffu, c.b, lo);
  const uint32_t se = __shfl_sync(0xffffffffu, c.excl, lo);
  return sb + (t - se);
}

// Squared distance below which a candidate is certainly nearer than every point outside the block of Chebyshev radius r
// around c0.  Every point binned outside the block lies beyond one of its faces as grid_face places them (grid_cell_of's
// invariant), so its true distance to q exceeds the exact q - face gap along that axis.  The shrink covers only the
// rounding of that subtraction (<= 2^-24 relative) and of the candidates' fp32 squared distances (a few ulp).
__device__ __forceinline__ float ring_bound(const GridMeta& m, int3 c0, int r, float qx, float qy, float qz, bool& all) {
  all = (c0.x - r <= 0 && c0.y - r <= 0 && c0.z - r <= 0 && c0.x + r >= m.nx - 1 && c0.y + r >= m.ny - 1 && c0.z + r >= m.nz - 1);
  float bound = FLT_MAX;
  if (c0.x - r > 0) bound = fminf(bound, __fsub_rn(qx, grid_face(m.ox, c0.x - r, m.cell)));
  if (c0.x + r < m.nx - 1) bound = fminf(bound, __fsub_rn(grid_face(m.ox, c0.x + r + 1, m.cell), qx));
  if (c0.y - r > 0) bound = fminf(bound, __fsub_rn(qy, grid_face(m.oy, c0.y - r, m.cell)));
  if (c0.y + r < m.ny - 1) bound = fminf(bound, __fsub_rn(grid_face(m.oy, c0.y + r + 1, m.cell), qy));
  if (c0.z - r > 0) bound = fminf(bound, __fsub_rn(qz, grid_face(m.oz, c0.z - r, m.cell)));
  if (c0.z + r < m.nz - 1) bound = fminf(bound, __fsub_rn(grid_face(m.oz, c0.z + r + 1, m.cell), qz));
  const float safe = __fsub_rn(__fmul_rn(fmaxf(bound, 0.f), 1.0f - 1e-5f), __fmul_rn(1e-6f, m.cell));
  return safe > 0.f ? __fmul_rn(__fmul_rn(safe, safe), 1.0f - 1e-5f) : -1.f;  // squared; -1: no conclusion possible yet
}

// k-NN, k <= 32.  On return lane i < kth holds the i-th nearest (d2, id), ordered by (d2, id); the other lanes
// hold (FLT_MAX, 0xffffffff).
__device__ __forceinline__ void grid_knn_warp(const GridView& g, float qx, float qy, float qz, int kth, uint32_t exclude,
                                              float& my_d2, uint32_t& my_id) {
  const int lane = threadIdx.x & 31;
  my_d2 = FLT_MAX;
  my_id = 0xffffffffu;
  if (g.n <= 0 || kth <= 0) return;
  const GridMeta m = *g.meta;
  const int3 c0 = grid_cell_of(m, qx, qy, qz);
  const int want = min(kth, g.n - (exclude != 0xffffffffu ? 1 : 0));
  if (want <= 0) return;

  auto offer = [&](float d, uint32_t id, bool valid) {  // every lane offers one candidate
    float thr_d = __shfl_sync(0xffffffffu, my_d2, kth - 1);
    uint32_t thr_i = __shfl_sync(0xffffffffu, my_id, kth - 1);
    bool cand = valid && (d < thr_d || (d == thr_d && id < thr_i));
    unsigned mask = __ballot_sync(0xffffffffu, cand);
    while (mask) {
      const int src = __ffs(mask) - 1;
      const float cd = __shfl_sync(0xffffffffu, d, src);
      const uint32_t ci = __shfl_sync(0xffffffffu, id, src);
      // sorted insertion across the lanes: entries ranking after the candidate shift up by one lane
      const bool greater = (my_d2 > cd) || (my_d2 == cd && my_id > ci);
      const float up_d = __shfl_up_sync(0xffffffffu, my_d2, 1);
      const uint32_t up_i = __shfl_up_sync(0xffffffffu, my_id, 1);
      const bool prev_greater = (__shfl_up_sync(0xffffffffu, (int)greater, 1) != 0) && lane > 0;
      if (greater) {
        my_d2 = prev_greater ? up_d : cd;
        my_id = prev_greater ? up_i : ci;
      }
      if (lane >= kth) {
        my_d2 = FLT_MAX;
        my_id = 0xffffffffu;
      }
      thr_d = __shfl_sync(0xffffffffu, my_d2, kth - 1);
      thr_i = __shfl_sync(0xffffffffu, my_id, kth - 1);
      cand = cand && (lane != src) && (d < thr_d || (d == thr_d && id < thr_i));
      mask = __ballot_sync(0xffffffffu, cand);
    }
  };

  bool finished = false;
  for (int r = 0; r <= kMaxRing && !finished; r++) {
    const int nslots = 2 * (2 * r + 1) * (2 * r + 1);
    for (int s0 = 0; s0 < nslots; s0 += 32) {
      const RingCursor c = ring_slots(g, m, c0, r, s0, lane);
      for (uint32_t t0 = 0; t0 < c.total; t0 += 32) {
        const uint32_t t = t0 + lane;
        const bool valid = t < c.total;
        const uint32_t idx = ring_element(c, valid ? t : 0);
        float d = FLT_MAX;
        uint32_t id = 0xffffffffu;
        if (valid) {
          const float4 p = g.pts[idx];
          id = __float_as_uint(p.w);
          d = dist2_nofma(p.x, p.y, p.z, qx, qy, qz);
        }
        offer(d, id, valid && id != exclude);
      }
    }
    bool all;
    const float lim = ring_bound(m, c0, r, qx, qy, qz, all);
    if (all) {
      finished = true;
    } else if (lim > 0.f) {
      const int cnt = __popc(__ballot_sync(0xffffffffu, lane < kth && my_d2 < lim));
      if (cnt >= want) finished = true;
    }
  }
  if (!finished) {  // far outside the occupied cells: exact linear scan of the whole cloud
    my_d2 = FLT_MAX;
    my_id = 0xffffffffu;
    for (int base = 0; base < g.n; base += 32) {
      const int i = base + lane;
      float d = FLT_MAX;
      uint32_t id = 0xffffffffu;
      if (i < g.n) {
        const float4 p = g.pts[i];
        id = __float_as_uint(p.w);
        d = dist2_nofma(p.x, p.y, p.z, qx, qy, qz);
      }
      offer(d, id, i < g.n && id != exclude);
    }
  }
}

// Nearest neighbour (k = 1): every lane keeps the best of the candidates it read, one argmin reduction per ring.
// Returns (d2, id) of the nearest point in all lanes ((FLT_MAX, 0xffffffff) for an empty cloud).
__device__ __forceinline__ void grid_nn_warp(const GridView& g, float qx, float qy, float qz, float& out_d2, uint32_t& out_id) {
  const int lane = threadIdx.x & 31;
  float bd = FLT_MAX;
  uint32_t bi = 0xffffffffu;
  out_d2 = bd;
  out_id = bi;
  if (g.n <= 0) return;
  const GridMeta m = *g.meta;
  const int3 c0 = grid_cell_of(m, qx, qy, qz);
  auto take = [&](float d, uint32_t id) {
    if (d < bd || (d == bd && id < bi)) {
      bd = d;
      bi = id;
    }
  };
  auto reduce = [&]() {
    float d = bd;
    uint32_t i = bi;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, d, o);
      const uint32_t oi = __shfl_xor_sync(0xffffffffu, i, o);
      if (od < d || (od == d && oi < i)) {
        d = od;
        i = oi;
      }
    }
    out_d2 = d;
    out_id = i;
  };
  bool finished = false;
  for (int r = 0; r <= kMaxRing && !finished; r++) {
    const int nslots = 2 * (2 * r + 1) * (2 * r + 1);
    for (int s0 = 0; s0 < nslots; s0 += 32) {
      const RingCursor c = ring_slots(g, m, c0, r, s0, lane);
      for (uint32_t t0 = 0; t0 < c.total; t0 += 32) {
        const uint32_t t = t0 + lane;
        const bool valid = t < c.total;
        const uint32_t idx = ring_element(c, valid ? t : 0);
        if (valid) {
          const float4 p = g.pts[idx];
          take(dist2_nofma(p.x, p.y, p.z, qx, qy, qz), __float_as_uint(p.w));
        }
      }
    }
    bool all;
    const float lim = ring_bound(m, c0, r, qx, qy, qz, all);
    reduce();
    if (all || (lim > 0.f && out_d2 < lim)) finished = true;
  }
  if (!finished) {
    bd = FLT_MAX;
    bi = 0xffffffffu;
    for (int i = lane; i < g.n; i += 32) {
      const float4 p = g.pts[i];
      take(dist2_nofma(p.x, p.y, p.z, qx, qy, qz), __float_as_uint(p.w));
    }
    reduce();
  }
}

// Slots of the whole 3x3x3 block around c0 (rings 0 and 1 together): cells are contiguous along x, so the block is 9
// contiguous candidate ranges, one per (z, y) row — one round of cell_start loads instead of one per ring.
__device__ __forceinline__ RingCursor block3_slots(const GridView& g, const GridMeta& m, int3 c0, int lane) {
  uint32_t b = 0, e = 0;
  if (lane < 9) {
    const int z = c0.z + lane / 3 - 1, y = c0.y + lane % 3 - 1;
    if (z >= 0 && z < m.nz && y >= 0 && y < m.ny) {
      const int base = (z * m.ny + y) * m.nx;
      b = g.cell_start[base + max(c0.x - 1, 0)];
      e = g.cell_start[base + min(c0.x + 1, m.nx - 1) + 1];
    }
  }
  const uint32_t len = e - b;
  uint32_t incl = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {  // full-width scan: ring_element searches the prefixes of all 32 lanes
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  RingCursor c;
  c.b = b;
  c.excl = incl - len;
  c.total = __shfl_sync(0xffffffffu, incl, 31);
  return c;
}

// Nearest neighbour of Q query points at once (same result as Q calls of grid_nn_warp): the searches of the Q queries are
// walked in lock step, so the cell-range loads and the candidate loads of all of them are in flight together — the search
// of one point is a chain of dependent L2 round trips with little work in between, and a warp that walks them one point at
// a time (align_lm_kernel runs 8 warps per SM) is latency bound.  The first pass takes rings 0 and 1 as one block
// (block3_slots) and applies ring 1's exact stopping criterion; a query that has met it is skipped from then on.
template <int Q>
__device__ __forceinline__ void grid_nn_warp_multi(const GridView& g, const GridMeta& m, const float (&qx)[Q], const float (&qy)[Q],
                                                   const float (&qz)[Q], float (&out_d2)[Q], uint32_t (&out_id)[Q]) {
  const int lane = threadIdx.x & 31;
  float bd[Q];
  uint32_t bi[Q];
#pragma unroll
  for (int q = 0; q < Q; q++) {
    bd[q] = FLT_MAX;
    bi[q] = 0xffffffffu;
    out_d2[q] = FLT_MAX;
    out_id[q] = 0xffffffffu;
  }
  if (g.n <= 0) return;
  int3 c0[Q];
#pragma unroll
  for (int q = 0; q < Q; q++) c0[q] = grid_cell_of(m, qx[q], qy[q], qz[q]);
  unsigned done = 0;  // warp-uniform bit per query
  constexpr unsigned kAll = (1u << Q) - 1u;

  auto scan = [&](RingCursor (&c)[Q]) {  // read the flattened candidate lists of all queries, 32 per query and round
    uint32_t tmax = 0;
#pragma unroll
    for (int q = 0; q < Q; q++) tmax = max(tmax, c[q].total);
    for (uint32_t t0 = 0; t0 < tmax; t0 += 32) {
      const uint32_t t = t0 + lane;
      float4 p[Q];
      bool valid[Q];
#pragma unroll
      for (int q = 0; q < Q; q++) {
        valid[q] = t < c[q].total;
        const uint32_t idx = ring_element(c[q], valid[q] ? t : 0);
        p[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid[q]) p[q] = g.pts[idx];
      }
#pragma unroll
      for (int q = 0; q < Q; q++) {
        if (valid[q]) {
          const float d = dist2_nofma(p[q].x, p[q].y, p[q].z, qx[q], qy[q], qz[q]);
          const uint32_t id = __float_as_uint(p[q].w);
          if (d < bd[q] || (d == bd[q] && id < bi[q])) {
            bd[q] = d;
            bi[q] = id;
          }
        }
      }
    }
  };
  auto settle = [&](int r) {  // warp argmin per query + the exact stopping criterion of ring r
#pragma unroll
    for (int q = 0; q < Q; q++) {
      if ((done >> q) & 1u) continue;
      bool all;
      const float lim = ring_bound(m, c0[q], r, qx[q], qy[q], qz[q], all);
      float d = bd[q];
      uint32_t i = bi[q];
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, d, o);
        const uint32_t oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (od < d || (od == d && oi < i)) {
          d = od;
          i = oi;
        }
      }
      out_d2[q] = d;
      out_id[q] = i;
      if (all || (lim > 0.f && d < lim)) done |= 1u << q;
    }
  };

  {
    RingCursor c[Q];
#pragma unroll
    for (int q = 0; q < Q; q++) c[q] = block3_slots(g, m, c0[q], lane);
    scan(c);
    settle(1);
  }
  for (int r = 2; r <= kMaxRing && done != kAll; r++) {
    const int nslots = 2 * (2 * r + 1) * (2 * r + 1);
    for (int s0 = 0; s0 < nslots; s0 += 32) {
      RingCursor c[Q];
#pragma unroll
      for (int q = 0; q < Q; q++) {
        c[q] = ring_slots(g, m, c0[q], r, s0, lane);
        if ((done >> q) & 1u) c[q].total = 0;
      }
      scan(c);
    }
    settle(r);
  }
#pragma unroll
  for (int q = 0; q < Q; q++)  // far outside the occupied cells: the single-query search ends in its exact linear scan
    if (!((done >> q) & 1u)) grid_nn_warp(g, qx[q], qy[q], qz[q], out_d2[q], out_id[q]);
}

}  // namespace gsicp
