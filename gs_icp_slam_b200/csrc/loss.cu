// Fused mapping loss (SURVEY.md §8f, row N2): masked L1 + 11x11 Gaussian-window SSIM on the colour image and L1 on the
// depth image, forward and backward, as two kernels instead of the ~50 element-wise / depthwise-conv launches the
// reference's PyTorch code issues per mapper iteration.
//
// Replaces (same arithmetic, same masking rules):
//   utils/loss_utils.py:17-20   l1_loss:  |x - gt|, zeroed where gt == 0, mean over ALL elements
//   utils/loss_utils.py:38-69   ssim/_ssim: x := where(gt != 0, x, 0); five zero-padded 11x11 depthwise convolutions
//                               (mu1, mu2, E[x^2], E[y^2], E[xy]), C1 = 0.01^2, C2 = 0.03^2, mean of the map
//   mp_Mapper.py:225-242        loss = (1-l)*L1 + l*(1-SSIM) + 0.1 * L1(depth/10, gt_depth/10)
//
// The Gaussian window is separable (loss_utils.py:27-36 builds the 2-D window as an outer product), so each convolution
// is a horizontal then a vertical 11-tap pass over a 26x26 tile held in shared memory.  Backward uses the three
// per-pixel partial-derivative maps the forward kernel leaves behind (d ssim / d mu1, / d E[x^2], / d E[xy]); their
// convolution with the same window gives d(mean ssim)/dx without ever materialising the 121-tap adjoint.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

#include "host_common.h"

namespace gsicp {

constexpr int kLossTile = 16;
constexpr int kWin = 11;
constexpr int kHalo = kWin / 2;
constexpr int kLossIn = kLossTile + 2 * kHalo;  // 26
constexpr int kLossThreads = 128;                // 104 threads work in the horizontal pass, 64 in the vertical one
constexpr int kLossCtasPerSm = 10;
// forward grid: kLossCtasPerSm persistent CTAs per SM walking (tile, channel) items; the partial-sum slots of the work
// buffer are sized for up to kLossMaxSms multiprocessors so that its size does not depend on the device
constexpr int kLossMaxSms = 256;
constexpr int kLossFwdCtas = kLossMaxSms * kLossCtasPerSm;

struct LossWindow {
  float w[kWin];
};

struct LossArgs {
  int H, W;
  const float* image;     // [3][H][W]
  const float* depth;     // [1][H][W]
  const float* gt_image;  // [3][H][W]
  const float* gt_depth;  // [1][H][W]
  float lambda_dssim, depth_weight, inv_dmax;
  int mask_by_depth;      // gt_image := gt_image * (gt_depth > 0)   (mp_Mapper.py:225-228)
  float* maps;            // [3 maps][3 channels][H][W]   (NULL in a loss-only call is not supported)
  float* ssim_map;        // optional [3][H][W]
  double* partial;        // [blocks][3]: sum ssim, sum masked |x-gt|, sum masked depth L1
  unsigned int* counter;
  float* loss;            // scalar
  float* parts;           // optional [3]: L1, SSIM, L1 depth
};

__device__ __forceinline__ float block_sum(float v, float* s_red) {
  // kLossThreads threads
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < kLossThreads / 32; w++) r += s_red[w];
  return r;  // valid in thread 0
}

// Work item = (16x16 pixel tile, z) with z = 0..2 the colour channels (SSIM + L1) and z = 3 the depth image (L1 only).
// The grid is a few CTAs per SM; each CTA walks items with a grid stride and keeps its three partial sums in registers,
// so the cross-CTA reduction (one fence + one same-address atomic per CTA) is paid ~600 times, not once per tile.
__global__ void __launch_bounds__(kLossThreads, kLossCtasPerSm)
mapping_loss_forward_kernel(LossArgs a, LossWindow win) {
  __shared__ float sx[kLossIn][kLossIn], sy[kLossIn][kLossIn];
  __shared__ float sh[5][kLossIn][kLossTile];
  __shared__ float s_red[kLossThreads / 32];
  const int tiles_x = (a.W + kLossTile - 1) / kLossTile, tiles_y = (a.H + kLossTile - 1) / kLossTile;
  const int items = tiles_x * tiles_y * 4;
  const size_t plane = (size_t)a.H * a.W;
  float s_ssim = 0.f, s_l1 = 0.f, s_d = 0.f;

  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int z = item / (tiles_x * tiles_y), t = item % (tiles_x * tiles_y);
    const int x0 = (t % tiles_x) * kLossTile, y0 = (t / tiles_x) * kLossTile;
    if (z == 3) {
#pragma unroll
      for (int p = threadIdx.x; p < kLossTile * kLossTile; p += kLossThreads) {
        const int px = x0 + p % kLossTile, py = y0 + p / kLossTile;
        if (px < a.W && py < a.H) {
          const float gd = a.gt_depth[(size_t)py * a.W + px] * a.inv_dmax;
          const float d = a.depth[(size_t)py * a.W + px] * a.inv_dmax;
          s_d += (gd != 0.f) ? fabsf(d - gd) : 0.f;
        }
      }
      continue;
    }
    const float* X = a.image + z * plane;
    const float* Y = a.gt_image + z * plane;
    __syncthreads();  // the previous item's readers of sx/sy/sh are done
    // the three loads of an element are independent (the masking is applied afterwards) and the loop is unrolled, so all
    // of a thread's global loads are in flight together: one DRAM latency per item instead of up to nine
#pragma unroll
    for (int it = 0; it < (kLossIn * kLossIn + kLossThreads - 1) / kLossThreads; it++) {
      const int i = threadIdx.x + it * kLossThreads;
      if (i < kLossIn * kLossIn) {
        const int ly = i / kLossIn, lx = i % kLossIn;
        const int gx = x0 + lx - kHalo, gy = y0 + ly - kHalo;
        float xv = 0.f, yv = 0.f, dv = 1.f;
        if (gx >= 0 && gx < a.W && gy >= 0 && gy < a.H) {
          const size_t o = (size_t)gy * a.W + gx;
          yv = Y[o];
          xv = X[o];
          if (a.mask_by_depth) dv = a.gt_depth[o];
        }
        if (!(dv > 0.f)) yv = 0.f;
        sx[ly][lx] = (yv != 0.f) ? xv : 0.f;  // ssim(): img = where(gt != 0, img, 0)
        sy[ly][lx] = yv;
      }
    }
    __syncthreads();
    // Horizontal pass, register sliding window: thread (row r, segment g) reads 14 consecutive inputs of row r once and
    // accumulates the 4 outputs 4g..4g+3 of the five windowed sums (26 rows x 4 segments = 104 threads; taps in order 0..10).
    if (threadIdx.x < kLossIn * 4) {
      const int r = threadIdx.x >> 2, c0 = (threadIdx.x & 3) * 4;
      float acc[5][4];
#pragma unroll
      for (int q = 0; q < 5; q++)
#pragma unroll
        for (int o = 0; o < 4; o++) acc[q][o] = 0.f;
#pragma unroll
      for (int i = 0; i < kWin + 3; i++) {
        const float xv = sx[r][c0 + i], yv = sy[r][c0 + i];
        const float xx = xv * xv, yy = yv * yv, xy = xv * yv;
#pragma unroll
        for (int o = 0; o < 4; o++) {
          const int k = i - o;
          if (k >= 0 && k < kWin) {
            const float w = win.w[k];
            acc[0][o] += w * xv;
            acc[1][o] += w * yv;
            acc[2][o] += w * xx;
            acc[3][o] += w * yy;
            acc[4][o] += w * xy;
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 5; q++)
#pragma unroll
        for (int o = 0; o < 4; o++) sh[q][r][c0 + o] = acc[q][o];
    }
    __syncthreads();
    // Vertical pass + SSIM: thread (column c, segment g) produces the 4 pixels (4g..4g+3, c) from 14 rows of `sh`.
    if (threadIdx.x < kLossTile * 4) {
      const int c = threadIdx.x & 15, r0 = (threadIdx.x >> 4) * 4;
      float acc[5][4];
#pragma unroll
      for (int q = 0; q < 5; q++)
#pragma unroll
        for (int o = 0; o < 4; o++) acc[q][o] = 0.f;
#pragma unroll
      for (int i = 0; i < kWin + 3; i++) {
        float v[5];
#pragma unroll
        for (int q = 0; q < 5; q++) v[q] = sh[q][r0 + i][c];
#pragma unroll
        for (int o = 0; o < 4; o++) {
          const int k = i - o;
          if (k >= 0 && k < kWin) {
            const float w = win.w[k];
#pragma unroll
            for (int q = 0; q < 5; q++) acc[q][o] += w * v[q];
          }
        }
      }
      const int px = x0 + c;
#pragma unroll
      for (int o = 0; o < 4; o++) {
        const int py = y0 + r0 + o;
        if (px < a.W && py < a.H) {
          const float mu1 = acc[0][o], mu2 = acc[1][o], exx = acc[2][o], eyy = acc[3][o], exy = acc[4][o];
          const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
          const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
          const float sig1 = exx - mu1_sq, sig2 = eyy - mu2_sq, sig12 = exy - mu12;
          const float A1 = 2.f * mu12 + C1, A2 = 2.f * sig12 + C2;
          const float B1 = mu1_sq + mu2_sq + C1, B2 = sig1 + sig2 + C2;
          const float inv = 1.f / (B1 * B2);
          const float ssim = (A1 * A2) * inv;
          s_ssim += ssim;
          // partial derivatives of ssim at this pixel w.r.t. its own mu1, E[x^2], E[xy] (E[.] = windowed means)
          const float d_mu1 = (2.f * mu2 * (A2 - A1)) * inv - ssim * (2.f * mu1 * (B2 - B1)) * inv;
          const float d_exx = -ssim / B2;
          const float d_exy = 2.f * A1 * inv;
          const size_t po = (size_t)py * a.W + px;
          a.maps[(0 * 3 + z) * plane + po] = d_mu1;
          a.maps[(1 * 3 + z) * plane + po] = d_exx;
          a.maps[(2 * 3 + z) * plane + po] = d_exy;
          if (a.ssim_map) a.ssim_map[z * plane + po] = ssim;
          // L1 term: sx holds the image where gt != 0 (and 0 elsewhere, where the term is masked anyway)
          const float yv = sy[r0 + o + kHalo][c + kHalo], xv = sx[r0 + o + kHalo][c + kHalo];
          s_l1 += (yv != 0.f) ? fabsf(xv - yv) : 0.f;
        }
      }
    }
  }
  // deterministic reduction: per-block partials, the last block adds them in index order
  const float b_ssim = block_sum(s_ssim, s_red);
  const float b_l1 = block_sum(s_l1, s_red);
  const float b_d = block_sum(s_d, s_red);
  const unsigned int nblocks = gridDim.x;
  const unsigned int bid = blockIdx.x;
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    a.partial[3 * (size_t)bid + 0] = (double)b_ssim;
    a.partial[3 * (size_t)bid + 1] = (double)b_l1;
    a.partial[3 * (size_t)bid + 2] = (double)b_d;
    __threadfence();
    s_last = (atomicAdd(a.counter, 1u) == nblocks - 1);
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    __shared__ double s_acc[3][kLossThreads / 32];
    double acc[3] = {0.0, 0.0, 0.0};
    for (unsigned int i = threadIdx.x; i < nblocks; i += blockDim.x) {
      acc[0] += a.partial[3 * (size_t)i + 0];
      acc[1] += a.partial[3 * (size_t)i + 1];
      acc[2] += a.partial[3 * (size_t)i + 2];
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_down_sync(0xffffffffu, acc[k], o);
      if ((threadIdx.x & 31) == 0) s_acc[k][threadIdx.x >> 5] = acc[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double t[3] = {0.0, 0.0, 0.0};
      for (int k = 0; k < 3; k++)
        for (int w = 0; w < kLossThreads / 32; w++) t[k] += s_acc[k][w];
      const double n3 = 3.0 * (double)a.H * (double)a.W, n1 = (double)a.H * (double)a.W;
      const float ssim = (float)(t[0] / n3), l1 = (float)(t[1] / n3), ld = (float)(t[2] / n1);
      *a.loss = (1.f - a.lambda_dssim) * l1 + a.lambda_dssim * (1.f - ssim) + a.depth_weight * ld;
      if (a.parts) {
        a.parts[0] = l1;
        a.parts[1] = ssim;
        a.parts[2] = ld;
      }
      *a.counter = 0u;  // ready for the next call
    }
  }
}

struct LossBwdArgs {
  int H, W;
  const float* image;
  const float* depth;
  const float* gt_image;
  const float* gt_depth;
  float lambda_dssim, depth_weight, inv_dmax;
  int mask_by_depth;
  const float* maps;
  const float* grad_loss;  // device scalar, NULL = 1
  float* grad_image;       // [3][H][W]
  float* grad_depth;       // [1][H][W]
};

__global__ void __launch_bounds__(kLossThreads)
mapping_loss_backward_kernel(LossBwdArgs a, LossWindow win) {
  __shared__ float sm[3][kLossIn][kLossIn];
  __shared__ float sh[3][kLossIn][kLossTile];
  const int x0 = blockIdx.x * kLossTile, y0 = blockIdx.y * kLossTile;
  const int z = blockIdx.z;
  const size_t plane = (size_t)a.H * a.W;
  const float up = a.grad_loss ? *a.grad_loss : 1.f;
  if (z == 3) {
#pragma unroll
    for (int p = threadIdx.x; p < kLossTile * kLossTile; p += kLossThreads) {
      const int px = x0 + p % kLossTile, py = y0 + p / kLossTile;
      if (px < a.W && py < a.H) {
        const size_t o = (size_t)py * a.W + px;
        const float gd = a.gt_depth[o] * a.inv_dmax, d = a.depth[o] * a.inv_dmax;
        const float diff = d - gd;
        const float sgn = (diff > 0.f) ? 1.f : ((diff < 0.f) ? -1.f : 0.f);
        a.grad_depth[o] = (gd != 0.f) ? up * a.depth_weight * sgn * a.inv_dmax / (float)plane : 0.f;
      }
    }
    return;
  }
#pragma unroll
  for (int it = 0; it < (kLossIn * kLossIn + kLossThreads - 1) / kLossThreads; it++) {
    const int i = threadIdx.x + it * kLossThreads;
    if (i < kLossIn * kLossIn) {
      const int ly = i / kLossIn, lx = i % kLossIn;
      const int gx = x0 + lx - kHalo, gy = y0 + ly - kHalo;
      const bool ok = gx >= 0 && gx < a.W && gy >= 0 && gy < a.H;
      const size_t o = ok ? (size_t)gy * a.W + gx : 0;
#pragma unroll
      for (int m = 0; m < 3; m++) sm[m][ly][lx] = ok ? a.maps[(m * 3 + z) * plane + o] : 0.f;
    }
  }
  __syncthreads();
  // separable convolution of the three partial maps with register sliding windows (see the forward kernel)
  if (threadIdx.x < kLossIn * 4) {
    const int r = threadIdx.x >> 2, c0 = (threadIdx.x & 3) * 4;
    float acc[3][4];
#pragma unroll
    for (int q = 0; q < 3; q++)
#pragma unroll
      for (int o = 0; o < 4; o++) acc[q][o] = 0.f;
#pragma unroll
    for (int i = 0; i < kWin + 3; i++) {
      const float v0 = sm[0][r][c0 + i], v1 = sm[1][r][c0 + i], v2 = sm[2][r][c0 + i];
#pragma unroll
      for (int o = 0; o < 4; o++) {
        const int k = i - o;
        if (k >= 0 && k < kWin) {
          const float w = win.w[k];
          acc[0][o] += w * v0;
          acc[1][o] += w * v1;
          acc[2][o] += w * v2;
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 3; q++)
#pragma unroll
      for (int o = 0; o < 4; o++) sh[q][r][c0 + o] = acc[q][o];
  }
  __syncthreads();
  if (threadIdx.x >= kLossTile * 4) return;
  const int c = threadIdx.x & 15, r0 = (threadIdx.x >> 4) * 4;
  float acc[3][4];
#pragma unroll
  for (int q = 0; q < 3; q++)
#pragma unroll
    for (int o = 0; o < 4; o++) acc[q][o] = 0.f;
#pragma unroll
  for (int i = 0; i < kWin + 3; i++) {
    const float v0 = sh[0][r0 + i][c], v1 = sh[1][r0 + i][c], v2 = sh[2][r0 + i][c];
#pragma unroll
    for (int o = 0; o < 4; o++) {
      const int k = i - o;
      if (k >= 0 && k < kWin) {
        const float w = win.w[k];
        acc[0][o] += w * v0;
        acc[1][o] += w * v1;
        acc[2][o] += w * v2;
      }
    }
  }
  const int qx = x0 + c;
  const float n3 = 3.f * (float)plane;
#pragma unroll
  for (int o = 0; o < 4; o++) {
    const int qy = y0 + r0 + o;
    if (qx >= a.W || qy >= a.H) continue;
    const size_t po = (size_t)qy * a.W + qx;
    float yv = a.gt_image[z * plane + po];
    if (a.mask_by_depth && !(a.gt_depth[po] > 0.f)) yv = 0.f;
    const float xr = a.image[z * plane + po];
    float g = 0.f;
    if (yv != 0.f) {
      const float dssim = (acc[0][o] + 2.f * xr * acc[1][o] + yv * acc[2][o]) / n3;  // d(mean ssim)/dx, x = image where gt != 0
      const float diff = xr - yv;
      const float sgn = (diff > 0.f) ? 1.f : ((diff < 0.f) ? -1.f : 0.f);
      g = (1.f - a.lambda_dssim) * sgn / n3 - a.lambda_dssim * dssim;
    }
    a.grad_image[z * plane + po] = up * g;
  }
}

static LossWindow make_window() {
  // loss_utils.py:27-29: gauss[x] = exp(-(x - 5)^2 / (2 * 1.5^2)), normalised; the reference evaluates it in Python floats
  // (double) and stores float32
  LossWindow w;
  double g[kWin], s = 0.0;
  for (int i = 0; i < kWin; i++) {
    g[i] = std::exp(-(double)((i - kHalo) * (i - kHalo)) / (2.0 * 1.5 * 1.5));
    s += (double)(float)g[i];
  }
  // torch.Tensor([...]) rounds each tap to float32 first, then `gauss / gauss.sum()` divides in float32
  float sf = 0.f;
  for (int i = 0; i < kWin; i++) sf += (float)g[i];
  (void)s;
  for (int i = 0; i < kWin; i++) w.w[i] = (float)g[i] / sf;
  return w;
}

}  // namespace gsicp

using namespace gsicp;

extern "C" {

size_t gsicp_mapping_loss_work_bytes(int H, int W) {
  if (H <= 0 || W <= 0) return 0;
  const size_t plane = (size_t)H * W;
  return 9 * plane * sizeof(float) + (size_t)kLossFwdCtas * 3 * sizeof(double) + 64;
}

static inline char* loss_partial_ptr(void* work, int H, int W) {
  const size_t plane = (size_t)H * W;
  size_t off = 9 * plane * sizeof(float);
  off = (off + 15) & ~size_t(15);
  return (char*)work + off;
}

int gsicp_mapping_loss_forward(int H, int W, const float* d_image, const float* d_depth, const float* d_gt_image,
                               const float* d_gt_depth, float lambda_dssim, float depth_weight, float d_max,
                               int mask_by_depth, float* d_loss, float* d_parts3, float* d_ssim_map, void* d_work, void* stream_) {
  if (H <= 0 || W <= 0 || !d_image || !d_depth || !d_gt_image || !d_gt_depth || !d_loss || !d_work || !(d_max > 0.f)) {
    set_error("gsicp_mapping_loss_forward: bad arguments");
    return GSICP_EINVAL;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  const int items = ((W + kLossTile - 1) / kLossTile) * ((H + kLossTile - 1) / kLossTile) * 4;
  const int ctas = std::min(device_sm_count(), kLossMaxSms) * kLossCtasPerSm;
  const int grid = items < ctas ? items : ctas;
  LossArgs a;
  a.H = H; a.W = W; a.image = d_image; a.depth = d_depth; a.gt_image = d_gt_image; a.gt_depth = d_gt_depth;
  a.lambda_dssim = lambda_dssim; a.depth_weight = depth_weight; a.inv_dmax = 1.f / d_max;
  a.mask_by_depth = mask_by_depth;
  a.maps = (float*)d_work; a.ssim_map = d_ssim_map;
  char* p = loss_partial_ptr(d_work, H, W);
  a.partial = (double*)p;
  a.counter = (unsigned int*)(p + (size_t)kLossFwdCtas * 3 * sizeof(double));
  a.loss = d_loss;
  a.parts = d_parts3;
  GSICP_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), stream));  // the work buffer is caller-allocated, not zeroed
  static const LossWindow win = make_window();
  ProfScope ps(kProfLossFwd, stream);
  GSICP_LAUNCH(mapping_loss_forward_kernel, grid, kLossThreads, 0, stream, a, win);
  GSICP_CUDA(cudaGetLastError());
  return GSICP_OK;
}

int gsicp_mapping_loss_backward(int H, int W, const float* d_image, const float* d_depth, const float* d_gt_image,
                                const float* d_gt_depth, float lambda_dssim, float depth_weight, float d_max,
                                int mask_by_depth, const float* d_grad_loss, const void* d_work, float* d_grad_image, float* d_grad_depth,
                                void* stream_) {
  if (H <= 0 || W <= 0 || !d_image || !d_depth || !d_gt_image || !d_gt_depth || !d_work || !d_grad_image || !d_grad_depth ||
      !(d_max > 0.f)) {
    set_error("gsicp_mapping_loss_backward: bad arguments");
    return GSICP_EINVAL;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  const dim3 grid((W + kLossTile - 1) / kLossTile, (H + kLossTile - 1) / kLossTile, 4);
  LossBwdArgs a;
  a.H = H; a.W = W; a.image = d_image; a.depth = d_depth; a.gt_image = d_gt_image; a.gt_depth = d_gt_depth;
  a.lambda_dssim = lambda_dssim; a.depth_weight = depth_weight; a.inv_dmax = 1.f / d_max;
  a.mask_by_depth = mask_by_depth;
  a.maps = (const float*)d_work; a.grad_loss = d_grad_loss; a.grad_image = d_grad_image; a.grad_depth = d_grad_depth;
  static const LossWindow win = make_window();
  ProfScope ps(kProfLossBwd, stream);
  GSICP_LAUNCH(mapping_loss_backward_kernel, grid, kLossThreads, 0, stream, a, win);
  GSICP_CUDA(cudaGetLastError());
  return GSICP_OK;
}

}  // extern "C"
