// Full-image evaluation scores of one rendered view against its held-out photograph (the `eval` command, nerfstudio
// ns-eval; DESIGN section 4.3o).  Everything stays on the device: the host reads one small record per image.
//   image_stats_kernel     one pass over the image: squared error of the clamped rgb, min / max of both images (SSIM's
//   stats_finish_kernel    data_range), the accumulation sum and the fruit confusion counts of sigmoid(logit) > 0.9
//                          against mask > 0.5 -- per-block partials, then one fixed-order finish
//   ssim_tile_kernel       torchmetrics' SSIM (11x11 gaussian window, sigma 1.5, k1 0.01, k2 0.03): one CTA per 32x16
//   ssim_finish_kernel     tile of the cropped map, the tile plus its 10-pixel apron staged in shared memory channel by
//                          channel, horizontal then vertical 11-tap passes, per-tile sums, one fixed-order finish
// torchmetrics reflect-pads both images by 5, filters, and crops 5 pixels off every side of the map before the mean.  A
// kept pixel's window therefore lies wholly inside the image and never touches a padded value, so the kernel filters the
// unpadded image over the (H - 10) x (W - 10) interior and needs no padding logic (tests/test_eval_host.py proves the
// equivalence against the padded torch version).
// The inputs are fp32; the squared error, the window sums and the SSIM formula are fp64, so image_metrics.
// restated_image_scores restates the kernels to rounding, and the fp32 torch path agrees to ~1e-6.  No floating-point
// atomics: each block combines its threads in a fixed tree and the finish kernels add the partials in index order, so
// repeated calls give identical bits.
#include <math_constants.h>
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kStatBlocks = FNR_IMAGE_STATS_PARTIALS;
constexpr int kStatFields = 10;  // the first ten record slots, in record order
constexpr int kWin = 11, kHalo = kWin / 2;
constexpr int kTileW = 32, kTileH = 16;
constexpr int kInW = kTileW + 2 * kHalo, kInH = kTileH + 2 * kHalo;

// torch.clamp(x, 0, 1): NaN stays NaN
__device__ __forceinline__ float clamp01(float x) { return x != x ? x : fminf(fmaxf(x, 0.f), 1.f); }

// Sum over the block in a fixed tree (xor shuffles, then warp 0 over the warp sums); the total is valid in thread 0.
__device__ __forceinline__ double block_sum(double v, double* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // s_warp may still be read from the previous call
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < kWarps ? s_warp[lane] : 0.0;
#pragma unroll
    for (int o = kWarps / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;
}

__device__ __forceinline__ float block_min(float v, float* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < kWarps ? s_warp[lane] : CUDART_INF_F;
#pragma unroll
    for (int o = kWarps / 2; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  }
  return v;
}

struct KStats {
  const float* rgb;        // [P,3] unclamped
  const float* semantics;  // [P] logits
  const float* accumulation;  // [P]
  const float* image;      // [P,3]
  const float* fruit_mask; // [P]
  long long P;
  double* partials;        // [kStatBlocks][kStatFields]
  double* record;
};

__global__ void __launch_bounds__(kThreads) image_stats_kernel(KStats A) {
  __shared__ double s_d[kWarps];
  __shared__ float s_f[kWarps];
  double sse = 0.0, acc = 0.0;
  float rlo = CUDART_INF_F, rhi = -CUDART_INF_F, ilo = CUDART_INF_F, ihi = -CUDART_INF_F;
  int tp = 0, fp = 0, fn = 0, tn = 0;  // a thread sees at most P / gridDim.x / 256 + 1 pixels
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < A.P; p += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const float c = clamp01(__ldg(A.rgb + 3 * p + q)), t = __ldg(A.image + 3 * p + q);
      const double d = (double)c - (double)t;
      sse += d * d;
      rlo = fminf(rlo, c);
      rhi = fmaxf(rhi, c);
      ilo = fminf(ilo, t);
      ihi = fmaxf(ihi, t);
    }
    acc += (double)__ldg(A.accumulation + p);
    // the thresholding FruitModel.get_outputs applies: fp32 sigmoid(logit) > 0.9
    const bool pred = 1.f / (1.f + expf(-__ldg(A.semantics + p))) > 0.9f;
    const bool truth = __ldg(A.fruit_mask + p) > 0.5f;
    tp += pred && truth;
    fp += pred && !truth;
    fn += !pred && truth;
    tn += !pred && !truth;
  }
  double* out = A.partials + (size_t)blockIdx.x * kStatFields;
  double v;
  float f;
  v = block_sum(sse, s_d);
  if (threadIdx.x == 0) out[0] = v;
  f = block_min(rlo, s_f);
  if (threadIdx.x == 0) out[1] = f;
  f = -block_min(-rhi, s_f);
  if (threadIdx.x == 0) out[2] = f;
  f = block_min(ilo, s_f);
  if (threadIdx.x == 0) out[3] = f;
  f = -block_min(-ihi, s_f);
  if (threadIdx.x == 0) out[4] = f;
  v = block_sum(acc, s_d);
  if (threadIdx.x == 0) out[5] = v;
  // counts are exact in fp64 (P < 2^31)
  v = block_sum((double)tp, s_d);
  if (threadIdx.x == 0) out[6] = v;
  v = block_sum((double)fp, s_d);
  if (threadIdx.x == 0) out[7] = v;
  v = block_sum((double)fn, s_d);
  if (threadIdx.x == 0) out[8] = v;
  v = block_sum((double)tn, s_d);
  if (threadIdx.x == 0) out[9] = v;
}

// lane k finishes field k over the blocks in index order
__global__ void stats_finish_kernel(const double* __restrict__ partials, int blocks, double* __restrict__ record) {
  const int k = threadIdx.x;
  if (k >= kStatFields) return;
  double v = partials[k];
  for (int b = 1; b < blocks; ++b) {
    const double x = partials[(size_t)b * kStatFields + k];
    v = (k == 1 || k == 3) ? fmin(v, x) : (k == 2 || k == 4) ? fmax(v, x) : v + x;
  }
  record[k] = v;
}

struct KSsim {
  const float* rgb;    // [H,W,3] unclamped
  const float* image;  // [H,W,3]
  int H, W;
  double window[kWin];  // normalised gaussian, fp64
  double* partials;     // one per tile, tiles in row-major order
  double* record;
};

// torchmetrics: data_range = max(preds.max() - preds.min(), target.max() - target.min()), the differences in fp32
__device__ __forceinline__ double record_data_range(const double* record) {
  const float a = __fsub_rn((float)record[FNR_REC_RGB_MAX], (float)record[FNR_REC_RGB_MIN]);
  const float b = __fsub_rn((float)record[FNR_REC_IMAGE_MAX], (float)record[FNR_REC_IMAGE_MIN]);
  return (double)fmaxf(a, b);
}

__global__ void __launch_bounds__(kThreads) ssim_tile_kernel(KSsim A) {
  __shared__ float s_x[kInH][kInW], s_y[kInH][kInW];
  __shared__ double s_h[5][kInH][kTileW];  // horizontal window sums of x, y, xx, yy, xy
  __shared__ double s_warp[kWarps];
  const int Ho = A.H - 2 * kHalo, Wo = A.W - 2 * kHalo;
  // output (oy, ox) of the cropped map is the window over input rows oy .. oy + 10, columns ox .. ox + 10
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const double range = record_data_range(A.record);
  const double c1 = (0.01 * range) * (0.01 * range), c2 = (0.03 * range) * (0.03 * range);
  double local = 0.0;
  for (int c = 0; c < 3; ++c) {
    for (int i = threadIdx.x; i < kInH * kInW; i += kThreads) {
      const int r = i / kInW, q = i - r * kInW;
      const int gy = y0 + r, gx = x0 + q;
      float x = 0.f, y = 0.f;
      if (gy < A.H && gx < A.W) {
        const size_t at = ((size_t)gy * A.W + gx) * 3 + c;
        x = clamp01(__ldg(A.rgb + at));
        y = __ldg(A.image + at);
      }
      s_x[r][q] = x;
      s_y[r][q] = y;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kInH * kTileW; i += kThreads) {
      const int r = i / kTileW, q = i - r * kTileW;
      double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
#pragma unroll
      for (int t = 0; t < kWin; ++t) {
        const double w = A.window[t], x = s_x[r][q + t], y = s_y[r][q + t];
        sx += w * x;
        sy += w * y;
        sxx += w * (x * x);
        syy += w * (y * y);
        sxy += w * (x * y);
      }
      s_h[0][r][q] = sx;
      s_h[1][r][q] = sy;
      s_h[2][r][q] = sxx;
      s_h[3][r][q] = syy;
      s_h[4][r][q] = sxy;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kTileH * kTileW; i += kThreads) {
      const int r = i / kTileW, q = i - r * kTileW;
      if (y0 + r >= Ho || x0 + q >= Wo) continue;
      double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int t = 0; t < kWin; ++t) {
        const double w = A.window[t];
#pragma unroll
        for (int k = 0; k < 5; ++k) m[k] += w * s_h[k][r + t][q];
      }
      const double mxx = m[0] * m[0], myy = m[1] * m[1], mxy = m[0] * m[1];
      const double vx = m[2] - mxx, vy = m[3] - myy, vxy = m[4] - mxy;
      local += ((2.0 * mxy + c1) * (2.0 * vxy + c2)) / ((mxx + myy + c1) * (vx + vy + c2));
    }
    // the next channel's loads only touch s_x / s_y, which no thread reads any more; its horizontal pass, which overwrites
    // s_h, starts after the barrier that follows those loads
  }
  const double total = block_sum(local, s_warp);
  if (threadIdx.x == 0) A.partials[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads) ssim_finish_kernel(const double* __restrict__ partials, long long tiles, double count,
                                                               double* __restrict__ record) {
  __shared__ double s_warp[kWarps];
  double v = 0.0;
  for (long long t = threadIdx.x; t < tiles; t += kThreads) v += partials[t];
  v = block_sum(v, s_warp);
  if (threadIdx.x == 0) {
    record[FNR_REC_SSIM] = v / count;
    record[FNR_REC_DATA_RANGE] = record_data_range(record);
  }
}

long long ssim_tiles(int H, int W) {
  if (H < kWin || W < kWin) return 0;
  return (long long)((H - 2 * kHalo + kTileH - 1) / kTileH) * ((W - 2 * kHalo + kTileW - 1) / kTileW);
}

size_t scratch_bytes_for(int H, int W) { return ((size_t)kStatBlocks * kStatFields + (size_t)ssim_tiles(H, W)) * sizeof(double); }

bool bad_size(const char* name, int32_t height, int32_t width) {
  if (height < 1 || width < 1 || (long long)height * width > 0x7fffffffLL / 3) {
    set_error("%s: image size %dx%d is not in 1 .. (2^31 - 1) / 3 pixels", name, width, height);
    return true;
  }
  return false;
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_image_metrics_scratch_bytes(int32_t height, int32_t width, size_t* bytes) {
  if (!bytes) {
    set_error("fnr_image_metrics_scratch_bytes: NULL bytes");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (bad_size("fnr_image_metrics_scratch_bytes", height, width)) return FNR_ERR_INVALID_ARGUMENT;
  *bytes = scratch_bytes_for(height, width);
  return FNR_OK;
}

int fnr_image_stats(const float* rgb, const float* semantics, const float* accumulation, const float* image, const float* fruit_mask,
                    int32_t height, int32_t width, void* scratch, size_t scratch_bytes, double* record, void* stream) {
  if (bad_size("fnr_image_stats", height, width)) return FNR_ERR_INVALID_ARGUMENT;
  if (!rgb || !semantics || !accumulation || !image || !fruit_mask || !scratch || !record || scratch_bytes < scratch_bytes_for(height, width)) {
    set_error("invalid arguments to fnr_image_stats (%dx%d): a NULL pointer, or %zu scratch bytes where %zu are needed", width, height,
              scratch_bytes, scratch_bytes_for(height, width));
    return FNR_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long P = (long long)height * width;
  KStats A{rgb, semantics, accumulation, image, fruit_mask, P, static_cast<double*>(scratch), record};
  const int blocks = grid_for(P, kThreads, kStatBlocks);  // a function of P alone: the partial sums do not depend on the device
  image_stats_kernel<<<blocks, kThreads, 0, st>>>(A);
  if (int rc = check_launch("image_stats_kernel")) return rc;
  stats_finish_kernel<<<1, 32, 0, st>>>(A.partials, blocks, record);
  return check_launch("stats_finish_kernel");
}

int fnr_ssim(const float* rgb, const float* image, int32_t height, int32_t width, void* scratch, size_t scratch_bytes, double* record,
             void* stream) {
  if (bad_size("fnr_ssim", height, width)) return FNR_ERR_INVALID_ARGUMENT;
  if (height < kWin || width < kWin) {
    set_error("fnr_ssim: a %dx%d image is smaller than the %dx%d window (the cropped SSIM map would be empty)", width, height, kWin, kWin);
    return FNR_ERR_UNSUPPORTED;
  }
  if (!rgb || !image || !scratch || !record || scratch_bytes < scratch_bytes_for(height, width)) {
    set_error("invalid arguments to fnr_ssim (%dx%d): a NULL pointer, or %zu scratch bytes where %zu are needed", width, height, scratch_bytes,
              scratch_bytes_for(height, width));
    return FNR_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  KSsim A{};
  A.rgb = rgb;
  A.image = image;
  A.H = height;
  A.W = width;
  // torchmetrics _gaussian(11, 1.5): exp(-(d / sigma)^2 / 2) over d = -5 .. 5, normalised
  double sum = 0.0;
  for (int t = 0; t < kWin; ++t) {
    const double d = (t - kHalo) / 1.5;
    A.window[t] = std::exp(-(d * d) / 2.0);
    sum += A.window[t];
  }
  for (int t = 0; t < kWin; ++t) A.window[t] /= sum;
  A.partials = static_cast<double*>(scratch) + (size_t)kStatBlocks * kStatFields;  // after fnr_image_stats' partials
  A.record = record;
  const int Ho = height - 2 * kHalo, Wo = width - 2 * kHalo;
  const dim3 grid((Wo + kTileW - 1) / kTileW, (Ho + kTileH - 1) / kTileH);
  if (grid.y > 65535u) {
    set_error("fnr_ssim: %d rows need more than 65535 tile rows", height);
    return FNR_ERR_UNSUPPORTED;
  }
  ssim_tile_kernel<<<grid, kThreads, 0, st>>>(A);
  if (int rc = check_launch("ssim_tile_kernel")) return rc;
  ssim_finish_kernel<<<1, kThreads, 0, st>>>(A.partials, ssim_tiles(height, width), 3.0 * (double)Ho * (double)Wo, record);
  return check_launch("ssim_finish_kernel");
}

}  // extern "C"
