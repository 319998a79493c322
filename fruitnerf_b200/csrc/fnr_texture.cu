// NeRF textures of exported meshes (nerfstudio texture_utils.export_textured_mesh with unwrap_method="custom"; DESIGN
// section 4.3p):
//   texel_rays_kernel      the per-face UV atlas in closed form: texel -> (face, barycentrics of the closest point of the
//                          face's UV triangle) -> one short ray from just outside the surface along the inverted normal
//   chart_rays_kernel      the same ray (texel_ray) for the owned texels of a chart atlas (fnr_unwrap.cu, DESIGN 4.3r)
//   mean_edge_partials     raylen = 2 * mean first-edge length: per-block fp64 sums over fixed face ranges, then one
//   mean_edge_finish       fixed-order finish (no atomics, so repeated calls give identical bits)
// The atlas layout is written out in include/fruitnerf_b200.h; fruitnerf_b200/texture.py restates both kernels.
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kEdgeBlocks = FNR_MEAN_EDGE_PARTIALS;

struct KTexelRays {
  const float* vertices;  // [V,3]
  const float* normals;   // [V,3]
  const int64_t* faces;   // [F,3]
  long long num_faces;
  int p, width, blocks_x;
  float half_len;          // 0.5 * raylen
  long long t0;
  int n;
  float* origins;     // [n,3]
  float* directions;  // [n,3]
};

__device__ __forceinline__ void load3(const float* a, int64_t i, float v[3]) {
  v[0] = a[3 * i];
  v[1] = a[3 * i + 1];
  v[2] = a[3 * i + 2];
}

// (w0 a + w1 b) + w2 c per component, every product and sum rounded (no FMA)
__device__ __forceinline__ void interp3(float w0, float w1, float w2, const float a[3], const float b[3], const float c[3], float out[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = __fadd_rn(__fadd_rn(__fmul_rn(w0, a[k]), __fmul_rn(w1, b[k])), __fmul_rn(w2, c[k]));
}

__device__ __forceinline__ float norm3(const float v[3]) {
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
}

// The ray of the surface point with barycentrics (w0, w1, w2) of face fv (texel_rays_kernel and chart_rays_kernel):
// position and normal interpolated in fp32 without FMA, the face normal where the interpolated one vanishes, then the
// origin 0.5 raylen outside the surface along the normal and the inverted normal as direction.
__device__ __forceinline__ void texel_ray(const float* vertices, const float* normals, const int64_t* fv, float w0, float w1, float w2,
                                          float half_len, float* origin, float* direction) {
  float v0[3], v1[3], v2[3], x[3], n[3];
  load3(vertices, fv[0], v0);
  load3(vertices, fv[1], v1);
  load3(vertices, fv[2], v2);
  interp3(w0, w1, w2, v0, v1, v2, x);
  {
    float n0[3], n1[3], n2[3];
    load3(normals, fv[0], n0);
    load3(normals, fv[1], n1);
    load3(normals, fv[2], n2);
    interp3(w0, w1, w2, n0, n1, n2, n);
  }
  float len = norm3(n);
  if (!(len > 1e-12f)) {  // vanishing (or NaN) interpolated normal: the right-hand face normal
    float e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      e1[k] = __fsub_rn(v1[k], v0[k]);
      e2[k] = __fsub_rn(v2[k], v0[k]);
    }
    n[0] = __fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1]));
    n[1] = __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2]));
    n[2] = __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]));
    len = norm3(n);
    if (!(len > 1e-12f)) {  // a degenerate face as well: +z
      n[0] = 0.f;
      n[1] = 0.f;
      n[2] = 1.f;
      len = 1.f;
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float nk = __fdiv_rn(n[k], len);
    origin[k] = __fadd_rn(x[k], __fmul_rn(half_len, nk));
    direction[k] = -nk;
  }
}

__global__ void __launch_bounds__(kThreads) texel_rays_kernel(KTexelRays A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const long long t = A.t0 + i;
  const int row = (int)(t / A.width), col = (int)(t % A.width);
  const int p = A.p, bw = p + 3;
  const int a = col % bw, b = row % p;
  const long long block = (long long)(row / p) * A.blocks_x + col / bw;
  const int half = a + b >= p + 1;
  const long long slot = 2 * block + half;
  const long long f = slot < A.num_faces ? slot : A.num_faces - 1;
  // the texel centre in its slot's frame, where the UV triangle is (0,0), (p-1,0), (0,p-1); its closest point (xs, ys)
  const int la = half ? p + 2 - a : a, lb = half ? p - 1 - b : b;
  float xs = (float)la, ys = (float)lb;
  if (la + lb > p - 1) {  // gutter: project onto the hypotenuse x + y = p - 1, clamped to its end points
    xs = fminf(fmaxf(xs - 0.5f, 0.f), (float)(p - 1));
    ys = (float)(p - 1) - xs;
  }
  const float pm1 = (float)(p - 1);
  const float s = __fdiv_rn(xs, pm1), u = __fdiv_rn(ys, pm1);
  const float w0 = __fsub_rn(__fsub_rn(1.f, s), u);
  texel_ray(A.vertices, A.normals, A.faces + 3 * f, w0, s, u, A.half_len, A.origins + 3 * (size_t)i, A.directions + 3 * (size_t)i);
}

// Rays of the owned texels of a chart atlas (fnr_chart_unwrap's compacted face and barycentrics per texel)
__global__ void __launch_bounds__(kThreads) chart_rays_kernel(const float* __restrict__ vertices, const float* __restrict__ normals,
                                                              const int64_t* __restrict__ faces, const int32_t* __restrict__ texel_faces,
                                                              const float* __restrict__ barycentrics, long long t0, int n, float half_len,
                                                              float* __restrict__ origins, float* __restrict__ directions) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long t = t0 + i;
  const float* w = barycentrics + 3 * t;
  texel_ray(vertices, normals, faces + 3 * (long long)texel_faces[t], w[0], w[1], w[2], half_len, origins + 3 * (size_t)i,
            directions + 3 * (size_t)i);
}

// Sum over the block in a fixed tree (xor shuffles, then warp 0 over the warp sums); the total is valid in thread 0.
__device__ __forceinline__ double block_sum(double v, double* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < kWarps ? s_warp[lane] : 0.0;
#pragma unroll
    for (int o = kWarps / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;
}

// block b sums |v1 - v0| over faces [b * per, min((b + 1) * per, F)), each thread its strided faces in order
__global__ void __launch_bounds__(kThreads) mean_edge_partials(const float* vertices, const int64_t* faces, long long F, long long per,
                                                               double* partials) {
  __shared__ double s_warp[kWarps];
  const long long lo = (long long)blockIdx.x * per, hi = lo + per < F ? lo + per : F;
  double acc = 0.0;
  for (long long f = lo + threadIdx.x; f < hi; f += kThreads) {
    const int64_t i0 = faces[3 * f], i1 = faces[3 * f + 1];
    double d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = __dsub_rn((double)vertices[3 * i1 + k], (double)vertices[3 * i0 + k]);
    acc = __dadd_rn(acc, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]))));
  }
  acc = block_sum(acc, s_warp);
  if (threadIdx.x == 0) partials[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(kThreads) mean_edge_finish(long long F, double* out) {
  __shared__ double s_warp[kWarps];
  double v = block_sum(out[1 + threadIdx.x], s_warp);  // kThreads == kEdgeBlocks
  if (threadIdx.x == 0) out[0] = v / (double)F;
}

static_assert(kThreads == kEdgeBlocks, "mean_edge_finish reads one partial per thread");

}  // namespace

// Atlas of F faces at p texels per triangle (the header's layout): blocks per row and the texture size
static bool atlas_layout(long long F, int p, long long* blocks_x, long long* width, long long* height) {
  if (F < 1 || F > FNR_TEXTURE_MAX_FACES || p < 2 || p > FNR_TEXTURE_MAX_SIDE) return false;
  const long long nb = (F + 1) / 2, need = nb * p, bw = p + 3;
  long long bx = (long long)std::ceil(std::sqrt((double)need / (double)bw));
  if (bx < 1) bx = 1;
  while (bx > 1 && (bx - 1) * (bx - 1) * bw >= need) --bx;
  while (bx * bx * bw < need) ++bx;
  *blocks_x = bx;
  *width = bx * bw;
  *height = (nb + bx - 1) / bx * p;
  return true;
}

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_texture_atlas_size(int64_t num_faces, int32_t px_per_uv_triangle, int64_t* width, int64_t* height) {
  long long bx, w, h;
  if (!width || !height || !atlas_layout(num_faces, px_per_uv_triangle, &bx, &w, &h)) {
    set_error("invalid arguments to fnr_texture_atlas_size (%lld faces, %d px per uv triangle)", (long long)num_faces, px_per_uv_triangle);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  *width = w;
  *height = h;
  return FNR_OK;
}

int fnr_texel_rays(const float* vertices, const float* normals, const int64_t* faces, int64_t num_faces, int32_t px_per_uv_triangle,
                   int32_t width, int32_t height, float raylen, int64_t texel_start, int32_t num_texels, float* origins, float* directions,
                   void* stream) {
  long long bx, w, h;
  if (!vertices || !normals || !faces || !origins || !directions) {
    set_error("fnr_texel_rays: NULL pointer");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (!atlas_layout(num_faces, px_per_uv_triangle, &bx, &w, &h)) {
    set_error("fnr_texel_rays: needs num_faces >= 1 and 2 <= px_per_uv_triangle <= %d, got %lld faces and %d", FNR_TEXTURE_MAX_SIDE,
              (long long)num_faces, px_per_uv_triangle);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (w != width || h != height || w > FNR_TEXTURE_MAX_SIDE || h > FNR_TEXTURE_MAX_SIDE) {
    set_error("fnr_texel_rays: the atlas of %lld faces at %d px per uv triangle is %lldx%lld (at most %d a side), got %dx%d",
              (long long)num_faces, px_per_uv_triangle, w, h, FNR_TEXTURE_MAX_SIDE, width, height);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_texels < 0 || texel_start < 0 || texel_start + num_texels > w * h || !(raylen > 0.f) || !std::isfinite(raylen)) {
    set_error("fnr_texel_rays: texels [%lld, %lld) of %lld, raylen %g", (long long)texel_start, (long long)texel_start + num_texels, w * h,
              (double)raylen);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_texels == 0) return FNR_OK;
  KTexelRays A{vertices, normals, faces, num_faces, px_per_uv_triangle, width, (int)bx, 0.5f * raylen, texel_start, num_texels,
               origins, directions};
  texel_rays_kernel<<<(num_texels + kThreads - 1) / kThreads, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A);
  return check_launch("texel_rays_kernel");
}

int fnr_chart_texel_rays(const float* vertices, const float* normals, const int64_t* faces, int64_t num_faces, const int32_t* texel_faces,
                         const float* barycentrics, int64_t num_owned, float raylen, int64_t texel_start, int32_t num_texels, float* origins,
                         float* directions, void* stream) {
  if (!vertices || !normals || !faces || !texel_faces || !barycentrics || !origins || !directions) {
    set_error("fnr_chart_texel_rays: NULL pointer");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_faces < 1 || num_texels < 0 || texel_start < 0 || texel_start + num_texels > num_owned || !(raylen > 0.f) || !std::isfinite(raylen)) {
    set_error("fnr_chart_texel_rays: %lld faces, texels [%lld, %lld) of %lld owned, raylen %g", (long long)num_faces, (long long)texel_start,
              (long long)texel_start + num_texels, (long long)num_owned, (double)raylen);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_texels == 0) return FNR_OK;
  chart_rays_kernel<<<(num_texels + kThreads - 1) / kThreads, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      vertices, normals, faces, texel_faces, barycentrics, texel_start, num_texels, 0.5f * raylen, origins, directions);
  return check_launch("chart_rays_kernel");
}

int fnr_mesh_mean_edge(const float* vertices, const int64_t* faces, int64_t num_faces, double* out, void* stream) {
  if (!vertices || !faces || !out || num_faces < 1) {
    set_error("invalid arguments to fnr_mesh_mean_edge (%lld faces)", (long long)num_faces);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long per = (num_faces + kEdgeBlocks - 1) / kEdgeBlocks;
  mean_edge_partials<<<kEdgeBlocks, kThreads, 0, st>>>(vertices, faces, num_faces, per, out + 1);
  if (int rc = check_launch("mean_edge_partials")) return rc;
  mean_edge_finish<<<1, kThreads, 0, st>>>(num_faces, out);
  return check_launch("mean_edge_finish");
}

}  // extern "C"
