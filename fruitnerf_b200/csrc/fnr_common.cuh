// Shared device helpers of the FruitNeRF hot path.
//
// Index-defining arithmetic (sample position -> [0,1]^3 -> per-level cell -> hash row) is written
// with explicit round-to-nearest intrinsics in the op order of the reference
// (fruit_nerf/fruit_field.py:170-179 and nerfstudio 0.3.2 Frustums.get_positions /
// SceneContraction / HashEncoding.pytorch_fwd) so that hash rows are bit-identical to the oracle;
// no FMA contraction can occur on those values.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/fruitnerf_b200.h"

namespace fnr {

constexpr uint32_t kPrimeY = 2654435761u;
constexpr uint32_t kPrimeZ = 805459861u;

struct Vec3 {
  float x, y, z;
};

// [NS] Frustums.get_positions: o + d * (start + end) / 2
__device__ __forceinline__ float sample_axis(float o, float d, float tsum) {
  return __fadd_rn(o, __fmul_rn(__fmul_rn(d, tsum), 0.5f));
}

// Returns the masked position in [0,1]^3 and the selector (fruit_field.py:170-179).
__device__ __forceinline__ Vec3 field_position(const float* __restrict__ o, const float* __restrict__ d, float start,
                                               float end, int position_mode, const float* __restrict__ aabb,
                                               bool& selector, Vec3* world = nullptr) {
  const float tsum = __fadd_rn(start, end);
  Vec3 p;
  p.x = sample_axis(o[0], d[0], tsum);
  p.y = sample_axis(o[1], d[1], tsum);
  p.z = sample_axis(o[2], d[2], tsum);
  if (world) *world = p;
  if (position_mode == FNR_POS_CONTRACT) {
    // [NS] SceneContraction(order=inf): where(mag < 1, x, (2 - 1/mag) * (x / mag))
    const float mag = fmaxf(fabsf(p.x), fmaxf(fabsf(p.y), fabsf(p.z)));
    if (!(mag < 1.0f)) {
      const float s = __fsub_rn(2.0f, __fdiv_rn(1.0f, mag));
      p.x = __fmul_rn(s, __fdiv_rn(p.x, mag));
      p.y = __fmul_rn(s, __fdiv_rn(p.y, mag));
      p.z = __fmul_rn(s, __fdiv_rn(p.z, mag));
    }
    p.x = __fmul_rn(__fadd_rn(p.x, 2.0f), 0.25f);  // (x + 2) / 4
    p.y = __fmul_rn(__fadd_rn(p.y, 2.0f), 0.25f);
    p.z = __fmul_rn(__fadd_rn(p.z, 2.0f), 0.25f);
  } else {
    // [NS] SceneBox.get_normalized_positions: (x - aabb[0]) / (aabb[1] - aabb[0])
    p.x = __fdiv_rn(__fsub_rn(p.x, aabb[0]), __fsub_rn(aabb[3], aabb[0]));
    p.y = __fdiv_rn(__fsub_rn(p.y, aabb[1]), __fsub_rn(aabb[4], aabb[1]));
    p.z = __fdiv_rn(__fsub_rn(p.z, aabb[2]), __fsub_rn(aabb[5], aabb[2]));
  }
  selector = (p.x > 0.0f) && (p.x < 1.0f) && (p.y > 0.0f) && (p.y < 1.0f) && (p.z > 0.0f) && (p.z < 1.0f);
  if (!selector) {
    p.x = 0.0f;
    p.y = 0.0f;
    p.z = 0.0f;
  }
  return p;
}

// One level of [NS] HashEncoding.pytorch_fwd: floor / ceil cell, offsets and the partial hashes.
struct LevelCell {
  uint32_t hx[2], hy[2], hz[2];  // [0] = floor, [1] = ceil, already multiplied by the primes
  float ox, oy, oz;              // scaled - floor
};

__device__ __forceinline__ LevelCell level_cell(const Vec3& p, float scale) {
  LevelCell c;
  const float sx = __fmul_rn(p.x, scale), sy = __fmul_rn(p.y, scale), sz = __fmul_rn(p.z, scale);
  const float fx = floorf(sx), fy = floorf(sy), fz = floorf(sz);
  c.ox = __fsub_rn(sx, fx);
  c.oy = __fsub_rn(sy, fy);
  c.oz = __fsub_rn(sz, fz);
  const uint32_t ix = (uint32_t)(int)fx, iy = (uint32_t)(int)fy, iz = (uint32_t)(int)fz;
  const uint32_t cx = (uint32_t)(int)ceilf(sx), cy = (uint32_t)(int)ceilf(sy), cz = (uint32_t)(int)ceilf(sz);
  c.hx[0] = ix;
  c.hx[1] = cx;
  c.hy[0] = iy * kPrimeY;
  c.hy[1] = cy * kPrimeY;
  c.hz[0] = iz * kPrimeZ;
  c.hz[1] = cz * kPrimeZ;
  return c;
}

// Corner order of the oracle / [NS]: 0 ccc, 1 cfc, 2 ffc, 3 fcc, 4 ccf, 5 cff, 6 fff, 7 fcf
// (x,y,z selectors; 1 = ceil).  kCornerSel[k] = x | y<<1 | z<<2.
__device__ __forceinline__ uint32_t corner_row(const LevelCell& c, int k, uint32_t mask, uint32_t level_base) {
  constexpr uint32_t sel[8] = {7u, 5u, 4u, 6u, 3u, 1u, 0u, 2u};
  const uint32_t s = sel[k];
  return ((c.hx[s & 1u] ^ c.hy[(s >> 1) & 1u] ^ c.hz[(s >> 2) & 1u]) & mask) + level_base;
}

// Trilinear weight of corner k (offset weights the CEIL corner, 1-offset the floor corner).
__device__ __forceinline__ float corner_weight(const LevelCell& c, int k) {
  constexpr uint32_t sel[8] = {7u, 5u, 4u, 6u, 3u, 1u, 0u, 2u};
  const uint32_t s = sel[k];
  const float wx = (s & 1u) ? c.ox : 1.0f - c.ox;
  const float wy = (s & 2u) ? c.oy : 1.0f - c.oy;
  const float wz = (s & 4u) ? c.oz : 1.0f - c.oz;
  return wx * wy * wz;
}

// Trilinear blend in the oracle's association order.
__device__ __forceinline__ float2 trilerp(const float2 (&f)[8], const LevelCell& c) {
  const float ox = c.ox, oy = c.oy, oz = c.oz;
  const float ix = 1.0f - ox, iy = 1.0f - oy, iz = 1.0f - oz;
  float2 f03, f12, f56, f47, a, b, r;
  f03.x = f[0].x * ox + f[3].x * ix;  f03.y = f[0].y * ox + f[3].y * ix;
  f12.x = f[1].x * ox + f[2].x * ix;  f12.y = f[1].y * ox + f[2].y * ix;
  f56.x = f[5].x * ox + f[6].x * ix;  f56.y = f[5].y * ox + f[6].y * ix;
  f47.x = f[4].x * ox + f[7].x * ix;  f47.y = f[4].y * ox + f[7].y * ix;
  a.x = f03.x * oy + f12.x * iy;      a.y = f03.y * oy + f12.y * iy;
  b.x = f47.x * oy + f56.x * iy;      b.y = f47.y * oy + f56.y * iy;
  r.x = a.x * oz + b.x * iz;          r.y = a.y * oz + b.y * iz;
  return r;
}

// [NS] components_from_spherical_harmonics(levels=4) on the shifted direction (d+1)/2.
__device__ __forceinline__ void sh_degree4(float dx, float dy, float dz, float* __restrict__ c) {
  const float x = (dx + 1.0f) * 0.5f, y = (dy + 1.0f) * 0.5f, z = (dz + 1.0f) * 0.5f;
  const float xx = x * x, yy = y * y, zz = z * z;
  c[0] = 0.28209479177387814f;
  c[1] = 0.4886025119029199f * y;
  c[2] = 0.4886025119029199f * z;
  c[3] = 0.4886025119029199f * x;
  c[4] = 1.0925484305920792f * x * y;
  c[5] = 1.0925484305920792f * y * z;
  c[6] = 0.9461746957575601f * zz - 0.31539156525251999f;
  c[7] = 1.0925484305920792f * x * z;
  c[8] = 0.5462742152960396f * (xx - yy);
  c[9] = 0.5900435899266435f * y * (3.0f * xx - yy);
  c[10] = 2.890611442640554f * x * y * z;
  c[11] = 0.4570457994644658f * y * (5.0f * zz - 1.0f);
  c[12] = 0.3731763325901154f * z * (5.0f * zz - 3.0f);
  c[13] = 0.4570457994644658f * x * (5.0f * zz - 1.0f);
  c[14] = 1.445305721320277f * z * (xx - yy);
  c[15] = 0.5900435899266435f * x * (xx - 3.0f * yy);
}

__device__ __forceinline__ float nan_to_num(float v) {
  if (v != v) return 0.0f;
  if (isinf(v)) return v > 0.0f ? 3.4028234663852886e38f : -3.4028234663852886e38f;
  return v;
}

__device__ __forceinline__ float sigmoidf_(float v) { return 1.0f / (1.0f + expf(-v)); }

// host-side error plumbing -------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
int check_launch(const char* what);  // after every <<<>>>: counts the launch, then cudaGetLastError

// Shape families the kernels are specialised for (SURVEY.md section 2.3).
//   SMALL: geo 15, semantic 15->64->64,        colour 63->64->64->3   (fruit_nerf)
//   BIG  : geo 30, semantic 30->128->128->64,  colour 78->64->64->3   (fruit_nerf_big / _huge)
enum Family { kFamilyNone = 0, kFamilySmall = 1, kFamilyBig = 2 };
Family classify(const fnr_field_desc* d);
int validate_desc(const fnr_field_desc* d);

}  // namespace fnr
