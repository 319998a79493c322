// Novel-view rendering of a trained model (the `render` command, nerfstudio ns-render):
//   camera_rays_kernel     Cameras.generate_rays for a pixel range of one frame of a camera set (perspective, fisheye,
//                          equirectangular; per-frame intrinsics; lens distortion), so a frame's rays are made chunk by
//                          chunk on the device
//   depth_range_kernel     per-block min / max of the depth outputs that take their near / far from the frame itself
//   compose_frame_kernel   _render_trajectory_video's per-frame image: apply_colormap / apply_depth_colormap of every
//                          requested output, concatenated side by side, quantised to uint8 as mediapy / PIL do
// All three are HBM-light: a few bytes per pixel next to the field evaluation of the same pixels.
#include <math_constants.h>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kRangeBlocks = FNR_COMPOSE_PARTIALS;

struct KCameraRays {
  const float* c2w;  // [F][3][4]
  const double *fx, *fy, *cx, *cy;  // [F]
  // lens cameras (fnr_camera_rays_lens): fp32 intrinsics in place of fx..cy, or all NULL
  const float *lens_fx, *lens_fy, *lens_cx, *lens_cy;  // [F]
  const float* distortion;  // [F,6] or NULL
  int frame, camera_type, height, width;
  long long p0;
  int n;
  float* origins;     // [n,3]
  float* directions;  // [n,3]
};

__global__ void __launch_bounds__(kThreads) camera_rays_kernel(KCameraRays A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const long long p = A.p0 + i;
  const int y = (int)(p / A.width), x = (int)(p % A.width);
  const float* m = A.c2w + 12 * (size_t)A.frame;  // [3][4] row-major
  float d[3];
  if (A.lens_fx) {
    // the training rays' arithmetic throughout (pixel_batch_kernel), so the ray of pixel (frame, y, x) is bit-identical to
    // the one a training batch draws for it
    const int f = A.frame;
    lens_direction(x, y, A.lens_fx[f], A.lens_fy[f], A.lens_cx[f], A.lens_cy[f], A.distortion ? A.distortion + 6 * (size_t)f : nullptr,
                   A.camera_type, d);
    world_ray(m, d, A.origins + 3 * (size_t)i, A.directions + 3 * (size_t)i);
    return;
  }
  // pixel centres: (u, v) = ((x + 0.5 - cx) / fx, -(y + 0.5 - cy) / fy) with python-float intrinsics, as torch's CUDA
  // kernels evaluate synthetic_scene.camera_rays: cx rounded to fp32 for the subtraction, the division a multiply by
  // fp32(1 / fx) formed in fp64
  const float cx = (float)A.cx[A.frame], cy = (float)A.cy[A.frame];
  const float ifx = (float)(1.0 / A.fx[A.frame]), ify = (float)(1.0 / A.fy[A.frame]);
  const float u = __fmul_rn(__fsub_rn(__fadd_rn((float)x, 0.5f), cx), ifx);
  const float v = -__fmul_rn(__fsub_rn(__fadd_rn((float)y, 0.5f), cy), ify);
  camera_direction(A.camera_type, u, v, d);
  // d = normalize(R d_cam) as synthetic_scene.camera_rays runs on the device: rounded products, and torch's reduction of a
  // 3-long row (two lanes: elements 0 and 2 in one, 1 in the other) sums them as (a0 + a2) + a1, for the rotation and the norm
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = __fadd_rn(__fadd_rn(__fmul_rn(m[4 * k], d[0]), __fmul_rn(m[4 * k + 2], d[2])), __fmul_rn(m[4 * k + 1], d[1]));
  const float nrm = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(w[0], w[0]), __fmul_rn(w[2], w[2])), __fmul_rn(w[1], w[1]))), 1e-12f);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    A.origins[3 * (size_t)i + k] = m[4 * k + 3];
    A.directions[3 * (size_t)i + k] = __fdiv_rn(w[k], nrm);
  }
}

// torch.min / torch.max: a NaN anywhere makes the result NaN
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || b != b) ? CUDART_NAN_F : fminf(a, b); }
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? CUDART_NAN_F : fmaxf(a, b); }

struct KCompose {
  int k, height, width;
  const float* images[FNR_MAX_FRAME_OUTPUTS];  // [H*W, channels]
  int kind[FNR_MAX_FRAME_OUTPUTS];
  int auto_range[FNR_MAX_FRAME_OUTPUTS];  // FNR_RANGE_AUTO_NEAR / _FAR: taken from this output's own min / max (`partials`)
  double near[FNR_MAX_FRAME_OUTPUTS], far[FNR_MAX_FRAME_OUTPUTS];
  const float* accumulation;              // [H*W] or NULL
  const float* turbo;                     // [256][3]
  float* partials;                        // [FNR_MAX_FRAME_OUTPUTS][kRangeBlocks][2]
  uint8_t* out;                           // [H][W*k][3]
};

// block b of output j: (min, max) of a grid-stride slice of the pixels
__global__ void __launch_bounds__(kThreads) depth_range_kernel(KCompose A) {
  __shared__ float s_lo[kThreads / 32], s_hi[kThreads / 32];
  const long long P = (long long)A.height * A.width;
  for (int j = 0; j < A.k; ++j) {
    if (!A.auto_range[j]) continue;
    float lo = CUDART_INF_F, hi = -CUDART_INF_F;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
      const float v = A.images[j][p];
      lo = nan_min(lo, v);
      hi = nan_max(hi, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
      s_lo[warp] = lo;
      s_hi[warp] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kThreads / 32; ++w) {
        lo = nan_min(lo, s_lo[w]);
        hi = nan_max(hi, s_hi[w]);
      }
      A.partials[((size_t)j * kRangeBlocks + blockIdx.x) * 2] = lo;
      A.partials[((size_t)j * kRangeBlocks + blockIdx.x) * 2 + 1] = hi;
    }
    __syncthreads();
  }
}

// mediapy to_uint8 / PIL: uint8(clip(x, 0, 1) * 255 + 0.5); NaN -> 0
__device__ __forceinline__ uint8_t quantise(float x) {
  x = x != x ? 0.f : fminf(fmaxf(x, 0.f), 1.f);
  return (uint8_t)(int)__fadd_rn(__fmul_rn(x, 255.f), 0.5f);
}

// nerfstudio apply_float_colormap: turbo[long(clip(nan_to_num(v, 0), 0, 1) * 255)]
__device__ __forceinline__ int turbo_index(float v) {
  v = v != v ? 0.f : fminf(fmaxf(v, 0.f), 1.f);
  return (int)__fmul_rn(v, 255.f);
}

__global__ void __launch_bounds__(kThreads) compose_frame_kernel(KCompose A) {
  __shared__ float s_near[FNR_MAX_FRAME_OUTPUTS], s_denom[FNR_MAX_FRAME_OUTPUTS];  // s_denom: fp32 reciprocal
  if (threadIdx.x < A.k) {
    const int j = threadIdx.x;
    double nr = A.near[j], fr = A.far[j];
    if (A.auto_range[j]) {
      float lo = CUDART_INF_F, hi = -CUDART_INF_F;
      for (int b = 0; b < kRangeBlocks; ++b) {
        lo = nan_min(lo, A.partials[((size_t)j * kRangeBlocks + b) * 2]);
        hi = nan_max(hi, A.partials[((size_t)j * kRangeBlocks + b) * 2 + 1]);
      }
      if (A.auto_range[j] & FNR_RANGE_AUTO_NEAR) nr = lo;
      if (A.auto_range[j] & FNR_RANGE_AUTO_FAR) fr = hi;
    }
    // (depth - near) / (far - near + 1e-10) with python-float near / far, as torch's CUDA kernels evaluate it: near
    // rounded to fp32 for the subtraction, the division a multiply by fp32(1 / (far - near + 1e-10)) formed in fp64
    s_near[j] = (float)nr;
    s_denom[j] = (float)(1.0 / (fr - nr + 1e-10));
  }
  __syncthreads();
  const long long P = (long long)A.height * A.width;
  const long long total = P * A.k;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    // t enumerates the output row-major: row y, column j * W + x
    const long long y = t / ((long long)A.width * A.k);
    const int col = (int)(t - y * A.width * A.k);
    const int j = col / A.width, x = col - j * A.width;
    const long long p = y * A.width + x;
    const float* img = A.images[j];
    float c[3];
    if (A.kind[j] == FNR_FRAME_COLOR) {
#pragma unroll
      for (int q = 0; q < 3; ++q) c[q] = img[3 * p + q];
    } else {
      float v = img[p];
      if (A.kind[j] == FNR_FRAME_DEPTH) v = __fmul_rn(__fsub_rn(v, s_near[j]), s_denom[j]);  // clipped with the turbo index
      const float* rgb = A.turbo + 3 * turbo_index(v);
#pragma unroll
      for (int q = 0; q < 3; ++q) c[q] = rgb[q];
      if (A.kind[j] == FNR_FRAME_DEPTH && A.accumulation) {
        // colored * accumulation + (1 - accumulation)
        const float a = A.accumulation[p], na = __fsub_rn(1.f, a);
#pragma unroll
        for (int q = 0; q < 3; ++q) c[q] = __fadd_rn(__fmul_rn(c[q], a), na);
      }
    }
    uint8_t* o = A.out + 3 * t;
#pragma unroll
    for (int q = 0; q < 3; ++q) o[q] = quantise(c[q]);
  }
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

static int camera_rays(const char* name, const KCameraRays& A, int32_t num_frames, int32_t camera_type, int32_t height, int32_t width,
                       int32_t frame, int64_t pixel_start, int32_t num_pixels, bool intrinsics, void* stream) {
  if (camera_type != FNR_CAMERA_PERSPECTIVE && camera_type != FNR_CAMERA_FISHEYE && camera_type != FNR_CAMERA_EQUIRECTANGULAR) {
    set_error("%s: unsupported camera_type %d", name, camera_type);
    return FNR_ERR_UNSUPPORTED;
  }
  if (num_frames < 1 || frame < 0 || frame >= num_frames || height < 1 || width < 1 || num_pixels < 0 || pixel_start < 0 ||
      pixel_start + num_pixels > (int64_t)height * width || (num_pixels > 0 && (!A.c2w || !intrinsics || !A.origins || !A.directions))) {
    set_error("invalid arguments to %s (frame %d of %d, %dx%d, pixels [%lld, %lld))", name, frame, num_frames, width, height,
              (long long)pixel_start, (long long)pixel_start + num_pixels);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_pixels == 0) return FNR_OK;
  camera_rays_kernel<<<(num_pixels + kThreads - 1) / kThreads, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A);
  return check_launch("camera_rays_kernel");
}

int fnr_camera_rays(const float* c2w, const double* fx, const double* fy, const double* cx, const double* cy, int32_t num_frames,
                    int32_t camera_type, int32_t height, int32_t width, int32_t frame, int64_t pixel_start, int32_t num_pixels,
                    float* origins, float* directions, void* stream) {
  KCameraRays A{c2w, fx, fy, cx, cy, nullptr, nullptr, nullptr, nullptr, nullptr, frame, camera_type, height, width, pixel_start, num_pixels,
                origins, directions};
  return camera_rays("fnr_camera_rays", A, num_frames, camera_type, height, width, frame, pixel_start, num_pixels, fx && fy && cx && cy, stream);
}

int fnr_camera_rays_lens(const float* c2w, const float* fx, const float* fy, const float* cx, const float* cy, const float* distortion,
                         int32_t num_frames, int32_t camera_type, int32_t height, int32_t width, int32_t frame, int64_t pixel_start,
                         int32_t num_pixels, float* origins, float* directions, void* stream) {
  if (!fx || !fy || !cx || !cy) {
    set_error("fnr_camera_rays_lens: NULL intrinsics");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KCameraRays A{c2w, nullptr, nullptr, nullptr, nullptr, fx, fy, cx, cy, distortion, frame, camera_type, height, width, pixel_start, num_pixels,
                origins, directions};
  return camera_rays("fnr_camera_rays_lens", A, num_frames, camera_type, height, width, frame, pixel_start, num_pixels, true, stream);
}

int fnr_compose_frame(const fnr_frame_output* outputs, int32_t num_outputs, const float* accumulation, int32_t height, int32_t width,
                      const float* turbo, float* scratch, uint8_t* image, void* stream) {
  if (!outputs || num_outputs < 1 || num_outputs > FNR_MAX_FRAME_OUTPUTS || height < 1 || width < 1 || !turbo || !image ||
      (long long)height * width * num_outputs > 0x7fffffffLL) {
    set_error("invalid arguments to fnr_compose_frame (%d outputs, %dx%d)", num_outputs, width, height);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KCompose A{};
  A.k = num_outputs;
  A.height = height;
  A.width = width;
  A.accumulation = accumulation;
  A.turbo = turbo;
  A.partials = scratch;
  A.out = image;
  bool any_auto = false;
  for (int j = 0; j < num_outputs; ++j) {
    const fnr_frame_output& o = outputs[j];
    if (!o.image || (o.kind != FNR_FRAME_COLOR && o.kind != FNR_FRAME_TURBO && o.kind != FNR_FRAME_DEPTH)) {
      set_error("fnr_compose_frame: output %d has no image or an unknown kind %d", j, o.kind);
      return FNR_ERR_INVALID_ARGUMENT;
    }
    A.images[j] = o.image;
    A.kind[j] = o.kind;
    A.auto_range[j] = o.kind == FNR_FRAME_DEPTH ? (o.auto_range & (FNR_RANGE_AUTO_NEAR | FNR_RANGE_AUTO_FAR)) : 0;
    A.near[j] = o.near_plane;
    A.far[j] = o.far_plane;
    any_auto |= A.auto_range[j] != 0;
  }
  if (any_auto && !scratch) {
    set_error("fnr_compose_frame: a depth output with auto_range needs scratch");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (any_auto) {
    depth_range_kernel<<<kRangeBlocks, kThreads, 0, st>>>(A);
    if (int rc = check_launch("depth_range_kernel")) return rc;
  }
  const long long total = (long long)height * width * num_outputs;
  compose_frame_kernel<<<grid_for(total, kThreads, sm_count() * 16), kThreads, 0, st>>>(A);
  return check_launch("compose_frame_kernel");
}

}  // extern "C"
