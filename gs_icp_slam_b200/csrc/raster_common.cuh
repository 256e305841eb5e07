// raster_common.cuh — shared types and per-Gaussian math of the H100 Gaussian-splat rasterizer.
//
// Data layout in HBM (DESIGN.md §3): every visible Gaussian is reduced by `preprocess` to ONE
// 48-byte "splat record" (3 x float4, 16-B aligned) that both render kernels read with three
// 128-bit loads per tile instance:
//   a = { px, py, conic_xx, conic_xy }      screen position, inverse 2D covariance
//   b = { conic_yy, opacity, cov_zx, cov_yz } ... and the z cross-covariances of the reference's float6
//   c = { r, g, b, view_depth }
// The reference keeps the same information in four separate arrays (float2 means2D, float6
// conic_opacity, float rgb[3], float depth: DGR/cuda_rasterizer/rasterizer_impl.h:30-45) and fetches
// rgb/depth from global memory once per contributing pixel-Gaussian pair (forward.cu:373-375,397).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gsicp {

constexpr int kTile = 16;            // reference BLOCK_X = BLOCK_Y = 16 (DGR/cuda_rasterizer/config.h:15-17)
constexpr int kTilePixels = kTile * kTile;

struct __align__(16) Splat {
  float4 a, b, c;
};

// Column-major 3x3 with the product evaluated as x0*y0 + x1*y1 + x2*y2 (left to right), the
// evaluation order the reference's matrix library uses, so that nvcc's fma contraction sees the
// same expression trees: radii and tile rectangles must come out bit-identical.
struct M3 {
  float m[3][3];  // m[col][row]
};

__device__ __forceinline__ M3 m3_mul(const M3& x, const M3& y) {
  M3 r;
#pragma unroll
  for (int c = 0; c < 3; c++) {
#pragma unroll
    for (int rr = 0; rr < 3; rr++) {
      r.m[c][rr] = x.m[0][rr] * y.m[c][0] + x.m[1][rr] * y.m[c][1] + x.m[2][rr] * y.m[c][2];
    }
  }
  return r;
}

__device__ __forceinline__ M3 m3_transpose(const M3& x) {
  M3 r;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int rr = 0; rr < 3; rr++) r.m[c][rr] = x.m[rr][c];
  return r;
}

// world -> view (rows 0..2 of the column-major 4x4 stored transposed; auxiliary.h:63-71)
__device__ __forceinline__ float3 xform_point_4x3(const float3 p, const float* __restrict__ mat) {
  return make_float3(mat[0] * p.x + mat[4] * p.y + mat[8] * p.z + mat[12],
                     mat[1] * p.x + mat[5] * p.y + mat[9] * p.z + mat[13],
                     mat[2] * p.x + mat[6] * p.y + mat[10] * p.z + mat[14]);
}

__device__ __forceinline__ float4 xform_point_4x4(const float3 p, const float* __restrict__ mat) {
  return make_float4(mat[0] * p.x + mat[4] * p.y + mat[8] * p.z + mat[12],
                     mat[1] * p.x + mat[5] * p.y + mat[9] * p.z + mat[13],
                     mat[2] * p.x + mat[6] * p.y + mat[10] * p.z + mat[14],
                     mat[3] * p.x + mat[7] * p.y + mat[11] * p.z + mat[15]);
}

// Rotation (un-normalised x,y,z,w quaternion — reference quirk, forward.cu:134-138) as the
// column-major matrix whose columns are the ROWS of the textbook rotation matrix.
__device__ __forceinline__ M3 quat_to_m3(float x, float y, float z, float w) {
  M3 R;
  R.m[0][0] = 1.f - 2.f * (y * y + z * z);
  R.m[0][1] = 2.f * (x * y - w * z);
  R.m[0][2] = 2.f * (x * z + w * y);
  R.m[1][0] = 2.f * (x * y + w * z);
  R.m[1][1] = 1.f - 2.f * (x * x + z * z);
  R.m[1][2] = 2.f * (y * z - w * x);
  R.m[2][0] = 2.f * (x * z - w * y);
  R.m[2][1] = 2.f * (y * z + w * x);
  R.m[2][2] = 1.f - 2.f * (x * x + y * y);
  return R;
}

// 3D covariance (upper triangle, 6 floats) from scale and rotation: Sigma = (S R)^T (S R)
// (forward.cu:122-168).
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 s, float mod, const float4 q, float* cov6) {
  M3 S;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int r = 0; r < 3; r++) S.m[c][r] = 0.f;
  S.m[0][0] = mod * s.x;
  S.m[1][1] = mod * s.y;
  S.m[2][2] = mod * s.z;
  const M3 R = quat_to_m3(q.x, q.y, q.z, q.w);
  const M3 Mx = m3_mul(S, R);
  const M3 Sg = m3_mul(m3_transpose(Mx), Mx);
  cov6[0] = Sg.m[0][0];
  cov6[1] = Sg.m[0][1];
  cov6[2] = Sg.m[0][2];
  cov6[3] = Sg.m[1][1];
  cov6[4] = Sg.m[1][2];
  cov6[5] = Sg.m[2][2];
}

// The EWA projection pieces shared by forward and backward (forward.cu:74-117, backward.cu:144-200):
// clamped view-space mean t, T = W*J, Vrk, and the 3x3 cov = T^T Vrk T (before the +0.3 low-pass).
struct Ewa {
  float3 t;          // clamped view-space position
  float txtz, tytz;  // unclamped ratios (backward needs them for the clamp mask)
  M3 T, Vrk, W, cov;
};

__device__ __forceinline__ Ewa ewa_project(const float3 mean, float fx, float fy, float tan_fovx, float tan_fovy,
                                           const float* cov3D, const float* __restrict__ view) {
  Ewa e;
  float3 t = xform_point_4x3(mean, view);
  const float limx = 1.3f * tan_fovx;
  const float limy = 1.3f * tan_fovy;
  e.txtz = t.x / t.z;
  e.tytz = t.y / t.z;
  t.x = fminf(limx, fmaxf(-limx, e.txtz)) * t.z;
  t.y = fminf(limy, fmaxf(-limy, e.tytz)) * t.z;
  e.t = t;

  M3 J;  // third row (0,0,1): the reference carries z through to obtain cov_zx / cov_yz
  J.m[0][0] = fx / t.z;  J.m[0][1] = 0.f;       J.m[0][2] = -(fx * t.x) / (t.z * t.z);
  J.m[1][0] = 0.f;       J.m[1][1] = fy / t.z;  J.m[1][2] = -(fy * t.y) / (t.z * t.z);
  J.m[2][0] = 0.f;       J.m[2][1] = 0.f;       J.m[2][2] = 1.f;

  e.W.m[0][0] = view[0]; e.W.m[0][1] = view[4]; e.W.m[0][2] = view[8];
  e.W.m[1][0] = view[1]; e.W.m[1][1] = view[5]; e.W.m[1][2] = view[9];
  e.W.m[2][0] = view[2]; e.W.m[2][1] = view[6]; e.W.m[2][2] = view[10];

  e.T = m3_mul(e.W, J);

  e.Vrk.m[0][0] = cov3D[0]; e.Vrk.m[0][1] = cov3D[1]; e.Vrk.m[0][2] = cov3D[2];
  e.Vrk.m[1][0] = cov3D[1]; e.Vrk.m[1][1] = cov3D[3]; e.Vrk.m[1][2] = cov3D[4];
  e.Vrk.m[2][0] = cov3D[2]; e.Vrk.m[2][1] = cov3D[4]; e.Vrk.m[2][2] = cov3D[5];

  e.cov = m3_mul(m3_mul(m3_transpose(e.T), e.Vrk), e.T);
  return e;
}

__device__ __forceinline__ float ndc_to_pix(float v, int S) {
  // double-precision constants in the reference (auxiliary.h:41-44): evaluated in fp64
  return (float)(((v + 1.0) * S - 1.0) * 0.5);
}

// Tile rectangle touched by a disc of integer radius (auxiliary.h:51-61).
__device__ __forceinline__ void tile_rect(float px, float py, int radius, int tiles_x, int tiles_y,
                                          int& x0, int& y0, int& x1, int& y1) {
  x0 = min(tiles_x, max(0, (int)((px - radius) / kTile)));
  y0 = min(tiles_y, max(0, (int)((py - radius) / kTile)));
  x1 = min(tiles_x, max(0, (int)((px + radius + kTile - 1) / kTile)));
  y1 = min(tiles_y, max(0, (int)((py + radius + kTile - 1) / kTile)));
}

// 16-byte asynchronous global -> shared copies (LDGSTS): the gather of the 48-B splat records into the staging ring does
// not pass through registers, so the loads of batch k+1 are in flight while batch k is blended.
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// Sub-tile culling shared by the forward and backward render kernels.
// A tile instance contributes to pixel p iff power(p) = -q(p - c) <= 0 and opacity * exp(power) >= 1/255, i.e.
// q(p - c) <= tau := ln(255 * opacity), with q(d) = 0.5 (A dx^2 + C dy^2) + B dx dy (the conic).  The warp's pixels lie
// in the rectangle [x0, x0+w] x [y0, y0+h]; q is convex, so its minimum over the rectangle is 0 if the centre is
// inside, else it is attained on the edge(s) facing the centre, where q restricted to the edge is a 1-D quadratic
// whose minimiser is clamped to the edge.  The instance is culled iff that exact minimum exceeds tau (plus a safety
// margin for fp32 rounding) — exactly the instances the reference skips for every pixel of the rectangle
// (forward.cu:359-366), so the blend is unchanged bit for bit.
__device__ __forceinline__ bool subtile_hit(const float4 a, const float4 b, float x0, float y0, float w, float h) {
  const float A = a.z, B = a.w, C = b.x, o = b.y;
  const float t255 = 255.f * o;
  if (!(t255 >= 0.999f)) return false;  // alpha = o * exp(power <= 0) can never reach 1/255
  if (!(A > 0.f && C > 0.f && A * C - B * B > 0.f)) return true;  // not an ellipse: do not cull
  const float tau = fmaxf(__logf(t255), 0.f) * 1.0005f + 2e-3f;
  const float cx = a.x, cy = a.y, x1 = x0 + w, y1 = y0 + h;
  const bool out_x = (cx < x0) || (cx > x1), out_y = (cy < y0) || (cy > y1);
  if (!out_x && !out_y) return true;
  float qmin = 3.0e38f;
  if (out_x) {
    const float dx = ((cx < x0) ? x0 : x1) - cx;
    const float ys = fminf(fmaxf(cy - (B / C) * dx, y0), y1);
    const float dy = ys - cy;
    qmin = 0.5f * (A * dx * dx + C * dy * dy) + B * dx * dy;
  }
  if (out_y) {
    const float dy = ((cy < y0) ? y0 : y1) - cy;
    const float xs = fminf(fmaxf(cx - (B / A) * dy, x0), x1);
    const float dx = xs - cx;
    qmin = fminf(qmin, 0.5f * (A * dx * dx + C * dy * dy) + B * dx * dy);
  }
  return qmin * 0.9995f <= tau;
}

__device__ const float kShC0 = 0.28209479177387814f;
__device__ const float kShC1 = 0.4886025119029199f;
__device__ const float kShC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                   -1.0925484305920792f, 0.5462742152960396f};
__device__ const float kShC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                   0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                   -0.5900435899266435f};

struct F3 {
  float x, y, z;
};
__device__ __forceinline__ F3 operator*(float s, F3 v) { return {s * v.x, s * v.y, s * v.z}; }
__device__ __forceinline__ F3 operator*(F3 v, float s) { return {v.x * s, v.y * s, v.z * s}; }
__device__ __forceinline__ F3 operator+(F3 a, F3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ F3 operator-(F3 a, F3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ float dot3(F3 a, F3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// Workspace sub-allocation: 128-B aligned carving of a byte buffer, like the reference's
// obtain() (rasterizer_impl.h:59-69) but with our own (smaller) state layout.
template <typename T>
__host__ inline T* carve(char*& p, size_t count) {
  uintptr_t u = (reinterpret_cast<uintptr_t>(p) + 127) & ~uintptr_t(127);
  T* r = reinterpret_cast<T*>(u);
  p = reinterpret_cast<char*>(r + count);
  return r;
}

struct GeomState {   // kept for backward: 97 B / Gaussian
  Splat* splats;     // [P]
  float* moments;    // [P][12] render-backward moments (raster_backward.cu); preprocess zeroes the rows of the visible
                     // Gaussians, the per-Gaussian backward kernel consumes and re-zeroes them: no P-sized fill launch
  uint8_t* clamped;  // [P] bit c set <=> SH colour channel c was clamped at 0
  static size_t bytes(size_t P) { return 3 * 128 + P * sizeof(Splat) + P * 12 * sizeof(float) + P; }
  static GeomState from(char* p, size_t P) {
    GeomState g;
    g.splats = carve<Splat>(p, P);
    g.moments = carve<float>(p, P * 12);
    g.clamped = carve<uint8_t>(p, P);
    return g;
  }
};

struct BinState {        // kept for backward: 5 B / tile instance
  uint32_t* point_list;  // [R] Gaussian index per tile instance, sorted by (tile, depth, index)
  // Sub-tile hit masks of the forward pass: for tile t, chunk c (list positions 32 c .. 32 c + 31 of the tile) and warp w
  // (the 8x4 sub-tile), bit i of hit[(hit_word(range.x, t) + c) * 8 + w] says whether instance 32 c + i survived the exact
  // sub-tile cull.  render_backward replays them instead of culling again.  Consecutive tiles never share a word.
  uint32_t* hit;
  static size_t hit_words(size_t R, size_t tiles) { return ((R >> 5) + tiles + 2) * 8; }
  static size_t bytes(size_t R, size_t tiles) { return 2 * 128 + (R ? R : 1) * sizeof(uint32_t) + hit_words(R, tiles) * sizeof(uint32_t); }
  static BinState from(char* p, size_t R, size_t tiles) {
    BinState b;
    b.point_list = carve<uint32_t>(p, R ? R : 1);
    b.hit = carve<uint32_t>(p, hit_words(R, tiles));
    return b;
  }
};
__host__ __device__ __forceinline__ size_t hit_word(uint32_t range_begin, int tile) { return (size_t)(range_begin >> 5) + (size_t)tile; }

struct ImgState {       // kept for backward: 8 B / pixel + 8 B / tile
  float* final_T;       // [N] transmittance after the last blended Gaussian (T == T_d, see DESIGN.md)
  uint32_t* n_contrib;  // [N] 1-based list position of the last blended Gaussian
  uint2* ranges;        // [tiles] [begin,end) into point_list
  uint32_t* tile_order; // [tiles] tile ids by decreasing instance count (launch order of the render CTAs)
  static size_t bytes(size_t N, size_t tiles) { return 4 * 128 + N * 8 + tiles * (sizeof(uint2) + 4); }
  static ImgState from(char* p, size_t N, size_t tiles) {
    ImgState s;
    s.final_T = carve<float>(p, N);
    s.n_contrib = carve<uint32_t>(p, N);
    s.ranges = carve<uint2>(p, tiles);
    s.tile_order = carve<uint32_t>(p, tiles);
    return s;
  }
};

}  // namespace gsicp
