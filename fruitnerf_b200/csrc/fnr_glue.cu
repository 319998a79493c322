// Small per-ray kernels around the fused field kernels -- the pieces of a training iteration that the reference
// spreads over dozens of elementwise / reduction launches:
//   pixel_batch_kernel     PixelSampler.sample + RayGenerator (fruit_nerf/data/fruit_datamanager.py:183-192; nerfstudio
//                          Cameras.generate_rays: a shared pinhole, or per-image intrinsics, lens distortion and the
//                          fisheye / equirectangular models): uniform (image, row, col) draws -> rays + targets
//   spaced_bins_kernel     SpacedSampler.generate_ray_samples: stratified bins in spacing space + the euclidean map
//                          (UniformLinDispPiecewiseSampler / UniformSampler; fruit_nerf/components/ray_samplers.py:54-104)
//   render_losses_kernel   MSELoss + BCEWithLogitsLoss(mean) + PSNR and their gradients (fruit_nerf.py:359-366, 396-399)
//   ray_metrics_kernel     nerfstudio distortion_loss on the final level (fruit_nerf.py:400) + median depth of a level
//                          (DepthRenderer(method="median"), fruit_nerf.py:339-340)
// All HBM-light (a few bytes per ray); they exist to take ~100 launches out of the iteration.
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) pixel_batch_kernel(KPixelBatch A) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < A.R; r += gridDim.x * blockDim.x) {
    // idx = floor(rand * [N, H, W]) (PixelSampler.sample_method), clamped against rand == 1 - ulp round-ups
    int ci = (int)floorf(__fmul_rn(A.rand[3 * r], (float)A.N));
    int y = (int)floorf(__fmul_rn(A.rand[3 * r + 1], (float)A.H));
    int x = (int)floorf(__fmul_rn(A.rand[3 * r + 2], (float)A.W));
    ci = min(ci, A.N - 1);
    y = min(y, A.H - 1);
    x = min(x, A.W - 1);
    const float* m = A.c2w + 12 * (size_t)ci;  // [3][4] row-major
    // pixel centres: d_cam = ((x + 0.5 - cx) / fx, -(y + 0.5 - cy) / fy, -1) for the pinhole; d = normalize(R d_cam)
    float dc[3];
    if (A.lens_fx) {
      lens_direction(x, y, A.lens_fx[ci], A.lens_fy[ci], A.lens_cx[ci], A.lens_cy[ci], A.distortion ? A.distortion + 6 * (size_t)ci : nullptr,
                     A.camera_type, dc);
    } else {
      dc[0] = __fdiv_rn(__fsub_rn(__fadd_rn((float)x, 0.5f), A.cx), A.fx);
      dc[1] = -__fdiv_rn(__fsub_rn(__fadd_rn((float)y, 0.5f), A.cy), A.fy);
      dc[2] = -1.0f;
    }
    world_ray(m, dc, A.origins + 3 * r, A.directions + 3 * r);
    A.camera_indices[r] = ci;
    if (A.indices) {
      A.indices[3 * (size_t)r] = ci;
      A.indices[3 * (size_t)r + 1] = y;
      A.indices[3 * (size_t)r + 2] = x;
    }
    const size_t px = ((size_t)ci * A.H + y) * A.W + x;
#pragma unroll
    for (int k = 0; k < 3; ++k) A.image[3 * r + k] = A.images[3 * px + k];
    A.fruit_mask[r] = A.masks[px];
  }
}

__device__ __forceinline__ float spacing_fn(int mode, float x) { return mode == 1 ? (x < 1.f ? __fdiv_rn(x, 2.f) : __fsub_rn(1.f, __fdiv_rn(1.f, __fmul_rn(2.f, x)))) : x; }
__device__ __forceinline__ float spacing_inv(int mode, float x) {
  return mode == 1 ? (x < 0.5f ? __fmul_rn(2.f, x) : __fdiv_rn(1.f, __fsub_rn(2.f, __fmul_rn(2.f, x)))) : x;
}

__global__ void __launch_bounds__(kThreads) spaced_bins_kernel(KSpacedBins A) {
  const long long total = (long long)A.R * (A.S + 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / (A.S + 1)), k = (int)(i % (A.S + 1));
    float b = A.base_bins[k];
    if (A.t_rand) {
      // centers = (b[1:] + b[:-1]) / 2 ; upper = [centers, b[-1]] ; lower = [b[0], centers] ; bins = lower + (upper - lower) * t
      const float lower = k == 0 ? A.base_bins[0] : __fdiv_rn(__fadd_rn(A.base_bins[k], A.base_bins[k - 1]), 2.0f);
      const float upper = k == A.S ? A.base_bins[A.S] : __fdiv_rn(__fadd_rn(A.base_bins[k + 1], A.base_bins[k]), 2.0f);
      const float t = A.t_rand[A.t_stride == 1 ? r : (size_t)r * (A.S + 1) + k];
      b = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t));
    }
    A.bins[i] = b;
    const float s_near = spacing_fn(A.mode, A.nears[r]), s_far = spacing_fn(A.mode, A.fars[r]);
    // spacing_to_euclidean_fn(x) = inv(x * s_far + (1 - x) * s_near)
    const float e = spacing_inv(A.mode, __fadd_rn(__fmul_rn(b, s_far), __fmul_rn(__fsub_rn(1.0f, b), s_near)));
    if (k < A.S) A.starts[(size_t)r * A.S + k] = e;
    if (k > 0) A.ends[(size_t)r * A.S + k - 1] = e;
  }
}

// One CTA: deterministic tree reduction over all rays (R is a few thousand).
__global__ void __launch_bounds__(1024) render_losses_kernel(KLosses A) {
  __shared__ float s_red[2][32];
  float se = 0.f, sb = 0.f;
  const float inv3r = 1.0f / (3.0f * (float)A.R), invr = 1.0f / (float)A.R;
  for (int r = threadIdx.x; r < A.R; r += blockDim.x) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float d = A.rgb[3 * r + k] - A.image[3 * r + k];
      se += d * d;
      if (A.d_rgb) A.d_rgb[3 * r + k] = 2.0f * d * inv3r;
    }
    const float x = A.semantics[r], y = A.fruit_mask[r];
    // BCEWithLogits: max(x, 0) - x*y + log1p(exp(-|x|))
    sb += fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
    if (A.d_semantics) A.d_semantics[r] = A.semantic_weight * (sigmoidf_(x) - y) * invr;
  }
  se = warp_sum(se);
  sb = warp_sum(sb);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_red[0][warp] = se;
    s_red[1][warp] = sb;
  }
  __syncthreads();
  if (warp == 0) {
    float a = lane < (blockDim.x >> 5) ? s_red[0][lane] : 0.f, b = lane < (blockDim.x >> 5) ? s_red[1][lane] : 0.f;
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) {
      const float mse = a * inv3r;
      A.out[0] = mse;
      A.out[1] = A.semantic_weight * b * invr;
      A.out[2] = -10.0f * log10f(mse);
    }
  }
}

// warp per ray.  mode bit 0: distortion (inter + intra) accumulated into *distortion (pre-zeroed) / R ;
// mode bit 1: median depth -> depth[r]
__global__ void __launch_bounds__(kThreads) ray_metrics_kernel(KRayMetrics A) {
  extern __shared__ float s_buf[];  // per warp: w[S], u[S]
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  float* w = s_buf + (size_t)wib * 2 * A.S;
  float* u = w + A.S;
  float block_acc = 0.f;
  for (int r = blockIdx.x * wpb + wib; r < A.R; r += gridDim.x * wpb) {
    const float* wr = A.weights + (size_t)r * A.S;
    if (A.distortion) {
      const float* t = A.sdist + (size_t)r * (A.S + 1);
      float intra = 0.f;
      for (int i = lane; i < A.S; i += 32) {
        const float wi = wr[i];
        w[i] = wi;
        u[i] = (t[i + 1] + t[i]) / 2;
        intra += wi * wi * (t[i + 1] - t[i]);
      }
      __syncwarp();
      float inter = 0.f;
      for (int i = lane; i < A.S; i += 32) {
        float acc = 0.f;
        const float ui = u[i];
        for (int j = 0; j < A.S; ++j) acc += w[j] * fabsf(ui - u[j]);
        inter += w[i] * acc;
      }
      const float tot = warp_sum(inter + intra / 3);
      if (lane == 0) block_acc += tot;
      __syncwarp();
    }
    if (A.depth) {
      float run = 0.f;
      int idx = A.S - 1;
      bool found = false;
      for (int c0 = 0; c0 < A.S && !found; c0 += 32) {
        const int i = c0 + lane;
        found = median_chunk(i < A.S ? wr[i] : 0.f, i < A.S, c0, lane, run, idx);
      }
      if (lane == 0) A.depth[r] = (A.starts[(size_t)r * A.S + idx] + A.ends[(size_t)r * A.S + idx]) / 2;
    }
  }
  if (A.distortion && lane == 0 && block_acc != 0.f) atomicAdd(A.distortion, block_acc / (float)A.R);
}

}  // namespace

int launch_pixel_batch(const KPixelBatch& A, cudaStream_t st) {
  if (A.R == 0) return FNR_OK;
  pixel_batch_kernel<<<(A.R + kThreads - 1) / kThreads, kThreads, 0, st>>>(A);
  return check_launch("pixel_batch_kernel");
}

int launch_spaced_bins(const KSpacedBins& A, cudaStream_t st) {
  const long long total = (long long)A.R * (A.S + 1);
  if (total == 0) return FNR_OK;
  spaced_bins_kernel<<<grid_for(total, kThreads, sm_count() * 8), kThreads, 0, st>>>(A);
  return check_launch("spaced_bins_kernel");
}

int launch_render_losses(const KLosses& A, cudaStream_t st) {
  render_losses_kernel<<<1, 1024, 0, st>>>(A);
  return check_launch("render_losses_kernel");
}

int launch_ray_metrics(const KRayMetrics& A, cudaStream_t st) {
  if (A.R == 0) return FNR_OK;
  const int wpb = kThreads / 32;
  const size_t smem = (size_t)wpb * 2 * A.S * sizeof(float);
  ray_metrics_kernel<<<grid_for(A.R, wpb, sm_count() * 4), kThreads, smem, st>>>(A);
  return check_launch("ray_metrics_kernel");
}

}  // namespace fnr
