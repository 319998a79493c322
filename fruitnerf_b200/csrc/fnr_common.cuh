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
#include <math_constants.h>
#include "../../include/fruitnerf_b200.h"

namespace fnr {

constexpr uint32_t kPrimeY = 2654435761u;
constexpr uint32_t kPrimeZ = 805459861u;
constexpr unsigned kFull = 0xffffffffu;  // every lane of a warp

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

// The two features of one hash-grid level at p: gather the cell's 8 corner rows (float2) and blend them.
__device__ __forceinline__ float2 level_gather(const float2* __restrict__ table, const Vec3& p, float scale, int level,
                                               uint32_t log2T) {
  const LevelCell c = level_cell(p, scale);
  const uint32_t mask = (1u << log2T) - 1u, base = (uint32_t)level << log2T;
  float2 f[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) f[k] = __ldg(table + corner_row(c, k, mask, base));
  return trilerp(f, c);
}

// Backward of level_gather: adds (g0, g1) times each corner's trilinear weight to the corner's gradient row.
__device__ __forceinline__ void level_scatter(float2* __restrict__ table_grad, const Vec3& p, float scale, int level,
                                              uint32_t log2T, float g0, float g1) {
  const LevelCell c = level_cell(p, scale);
  const uint32_t mask = (1u << log2T) - 1u, base = (uint32_t)level << log2T;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float w = corner_weight(c, k);
    if (w != 0.f) atomicAdd(table_grad + corner_row(c, k, mask, base), make_float2(w * g0, w * g1));
  }
}

// level_scatter of one level for the 32 points held by the lanes of a warp, with fewer reds.  When the lanes hold
// consecutive samples of a ray, neighbouring lanes often share a cell and so add to the same rows.  For each corner, lanes
// with equal rows in a row form a run; a segmented shuffle sum gives the run's total to its last lane, which alone issues
// the red.  A cell's floor-x and ceil-x corners differ in x only; with an even floor x their rows are r and r ^ 1 (the
// hash's x prime is 1 and the level base is even), one 16-byte-aligned pair, so where both runs end at the same lane their
// totals go out as one float4 red.  table_grad must be 16-byte aligned.
//
// All 32 lanes call this together from warp-uniform control flow, the same number of times: it shuffles and ballots with
// the full mask.  A lane with nothing to add passes active = false (its rows become the null key and its values zero).
__device__ __forceinline__ void warp_level_scatter(float2* __restrict__ table_grad, const LevelCell& c, bool active, int level,
                                                   uint32_t log2T, float g0, float g1, int lane) {
  constexpr uint32_t kNull = 0xffffffffu;
  constexpr int kCeilX[4] = {0, 1, 4, 5}, kFloorX[4] = {3, 2, 7, 6};  // x-neighbour corners in the oracle's order
  const uint32_t mask = (1u << log2T) - 1u, base = (uint32_t)level << log2T;
  active = active && (g0 != 0.f || g1 != 0.f);
  const uint32_t at_or_below = 0xffffffffu >> (31 - lane);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint32_t key[2];
    float v[2][2];
    int start[2];
    bool last[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = j ? kFloorX[q] : kCeilX[q];
      const float w = corner_weight(c, k);
      const bool on = active && w != 0.f;
      key[j] = on ? corner_row(c, k, mask, base) : kNull;
      v[j][0] = on ? w * g0 : 0.f;
      v[j][1] = on ? w * g1 : 0.f;
      const uint32_t up = __shfl_up_sync(kFull, key[j], 1);
      const uint32_t heads = __ballot_sync(kFull, lane == 0 || key[j] != up);
      start[j] = 31 - __clz(heads & at_or_below);
      last[j] = lane == 31 || ((heads >> (lane + 1)) & 1u);
    }
    // segmented inclusive sums: after the step of distance d, a lane holds the sum over its run's last 2d lanes.  The
    // loop ends when no lane with a row needs another step (a ballot, so every lane leaves on the same step).
    for (int d = 1; d < 32; d <<= 1) {
      const bool need0 = key[0] != kNull && lane - d >= start[0];
      const bool need1 = key[1] != kNull && lane - d >= start[1];
      if (!__ballot_sync(kFull, need0 || need1)) break;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float t0 = __shfl_up_sync(kFull, v[j][0], d), t1 = __shfl_up_sync(kFull, v[j][1], d);
        if (j ? need1 : need0) {
          v[j][0] += t0;
          v[j][1] += t1;
        }
      }
    }
    const bool red0 = last[0] && key[0] != kNull, red1 = last[1] && key[1] != kNull;
    if (red0 && red1 && (key[0] ^ key[1]) == 1u) {
      const bool lo0 = key[0] < key[1];
      const float4 v4 = lo0 ? make_float4(v[0][0], v[0][1], v[1][0], v[1][1]) : make_float4(v[1][0], v[1][1], v[0][0], v[0][1]);
      atomicAdd(reinterpret_cast<float4*>(table_grad + (key[0] & ~1u)), v4);
    } else {
      if (red0) atomicAdd(table_grad + key[0], make_float2(v[0][0], v[0][1]));
      if (red1) atomicAdd(table_grad + key[1], make_float2(v[1][0], v[1][1]));
    }
  }
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

// fp64 squared distance (dx*dx + dy*dy) + dz*dz with round-to-nearest intrinsics (no FMA): the numpy / scikit-learn order.
__device__ __forceinline__ double dist2(double ax, double ay, double az, double bx, double by, double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// ---- warp-per-ray primitives ----------------------------------------------------------------
// A ray's samples are walked in chunks of 32, lane i holding sample c0 + i; `run` arguments carry a sum over the
// earlier chunks.

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ float warp_incl_scan(float v, int lane) {  // sum over lanes <= lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(kFull, v, o);
    if (lane >= o) v += t;
  }
  return v;
}
__device__ __forceinline__ float warp_rev_incl_scan(float v, int lane) {  // sum over lanes >= lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_down_sync(kFull, v, o);
    if (lane + o < 32) v += t;
  }
  return v;
}

// Inclusive cumsum of value(i) over i < n: out(i, value(0) + ... + value(i)), the sum formed chunk by chunk.
template <class Value, class Out>
__device__ __forceinline__ void warp_cumsum(int n, int lane, Value value, Out out) {
  float run = 0.f;
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int i = c0 + lane;
    const float incl = warp_incl_scan(i < n ? value(i) : 0.f, lane);
    if (i < n) out(i, run + incl);
    run += __shfl_sync(kFull, incl, 31);
  }
}

// RaySamples.get_weights on one chunk: w_i = nan_to_num((1 - e^{-x_i}) e^{-X_i}), x = delta * sigma, X_i = sum_{j<i} x_j
// (0 for lanes past the ray's end, `in` false).  Adds the chunk's x to run_x.
__device__ __forceinline__ float chunk_weight(float x, bool in, int lane, float& run_x) {
  const float incl = warp_incl_scan(x, lane);
  // exclusive prefix by shuffle, not `incl - x`: an infinite sigma*delta must give T = 1 in front of it (torch.cumsum semantics)
  float excl = __shfl_up_sync(kFull, incl, 1);
  if (lane == 0) excl = 0.f;
  float w = 0.f;
  if (in) {
    const float alpha = 1.0f - expf(-x);
    const float T = expf(-(run_x + excl));
    w = nan_to_num(alpha * T);
  }
  run_x += __shfl_sync(kFull, incl, 31);
  return w;
}

// Backward of get_weights, with G_i = dL/dw_i:  dL/dx_j = G_j T_{j+1} - sum_{i>j} G_i w_i.  The suffix sums are formed
// from per-chunk totals and reverse scans, without the cancellation of "total - prefix" on long rays.
//
// sum of G_i w_i over the chunks after chunk ci, in lane ci (rays of at most 32 chunks); gw(i) = G_i w_i, i < S.
template <class GW>
__device__ __forceinline__ float later_chunks_sum(int S, int lane, GW gw) {
  float chunk_tot = 0.f;
  for (int c0 = 0, ci = 0; c0 < S; c0 += 32, ++ci) {
    const int i = c0 + lane;
    const float t = warp_sum(i < S ? gw(i) : 0.f);
    if (lane == ci) chunk_tot = t;
  }
  return warp_rev_incl_scan(chunk_tot, lane) - chunk_tot;
}
// sum_{k>i} G_k w_k for lane i of chunk ci: the in-chunk reverse scan plus the later chunks (later_chunks_sum)
__device__ __forceinline__ float chunk_suffix(float gw, float later_chunks, int ci, int lane) {
  return (warp_rev_incl_scan(gw, lane) - gw) + __shfl_sync(kFull, later_chunks, ci & 31);
}
// dL/dsigma_i = delta_i dL/dx_i; xin = the chunk's inclusive scan of x, so T_{i+1} = e^{-(run_x + xin)}
__device__ __forceinline__ float weights_dsigma(float delta, float G, float run_x, float xin, float suffix) {
  const float Tnext = expf(-(run_x + xin));
  return delta * (G * Tnext - suffix);
}

// DepthRenderer(method="median") on one chunk: searchsorted(cumsum(w), 0.5, side="left"), the first index whose
// cumulative weight is >= 0.5.  Returns true and sets `median` if it lies in this chunk; the caller starts `median` at
// S - 1, the clamp for rays whose weights never reach 0.5.  Adds the chunk's weight to run_w.
__device__ __forceinline__ bool median_chunk(float w, bool in, int c0, int lane, float& run_w, int& median) {
  const float wincl = warp_incl_scan(w, lane);
  const unsigned m = __ballot_sync(kFull, in && run_w + wincl >= 0.5f);
  run_w += __shfl_sync(kFull, wincl, 31);
  if (m) median = c0 + __ffs(m) - 1;
  return m != 0;
}

// camera model ------------------------------------------------------------------------------
// One definition of the lens for the training rays (pixel_batch_kernel) and the evaluation / render rays
// (camera_rays_kernel); DESIGN.md section 4.3j.

// [NS] camera_utils.radial_and_tangential_undistort(coords, [k1, k2, k3, k4, p1, p2], eps=1e-3, max_iterations=10):
// Newton's method on the OpenCV model, exactly 10 steps and no convergence test, a zero step where |det| <= eps.  Run in
// fp64 with every op rounded in the order of the expressions of data/camera_model.py, so that restatement reproduces it
// bit for bit; (u, v) are rounded back to fp32.
__device__ __forceinline__ void undistort_rt(const float* __restrict__ dist, float& u, float& v) {
  const double k1 = dist[0], k2 = dist[1], k3 = dist[2], k4 = dist[3], p1 = dist[4], p2 = dist[5];
  const double xd = u, yd = v;
  const double tp1 = __dmul_rn(2.0, p1), tp2 = __dmul_rn(2.0, p2), sp1 = __dmul_rn(6.0, p1), sp2 = __dmul_rn(6.0, p2);
  const double tk2 = __dmul_rn(2.0, k2), tk3 = __dmul_rn(3.0, k3);
  double x = xd, y = yd;
#pragma unroll 1
  for (int it = 0; it < 10; ++it) {
    const double r = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
    const double d = __dadd_rn(1.0, __dmul_rn(r, __dadd_rn(k1, __dmul_rn(r, __dadd_rn(k2, __dmul_rn(r, __dadd_rn(k3, __dmul_rn(r, k4))))))));
    const double x2 = __dmul_rn(2.0, x), y2 = __dmul_rn(2.0, y);
    // residuals: x d + 2 p1 x y + p2 (r + 2 x^2) - xd and y d + 2 p2 x y + p1 (r + 2 y^2) - yd
    const double fx = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(d, x), __dmul_rn(__dmul_rn(tp1, x), y)), __dmul_rn(p2, __dadd_rn(r, __dmul_rn(x2, x)))), xd);
    const double fy = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(d, y), __dmul_rn(__dmul_rn(tp2, x), y)), __dmul_rn(p1, __dadd_rn(r, __dmul_rn(y2, y)))), yd);
    // d'(r) = k1 + r (2 k2 + r (3 k3 + r 4 k4)) and the Jacobian of (fx, fy)
    const double d_r = __dadd_rn(k1, __dmul_rn(r, __dadd_rn(tk2, __dmul_rn(r, __dadd_rn(tk3, __dmul_rn(__dmul_rn(r, 4.0), k4))))));
    const double d_x = __dmul_rn(x2, d_r), d_y = __dmul_rn(y2, d_r);
    const double fx_x = __dadd_rn(__dadd_rn(__dadd_rn(d, __dmul_rn(d_x, x)), __dmul_rn(tp1, y)), __dmul_rn(sp2, x));
    const double fx_y = __dadd_rn(__dadd_rn(__dmul_rn(d_y, x), __dmul_rn(tp1, x)), __dmul_rn(tp2, y));
    const double fy_x = __dadd_rn(__dadd_rn(__dmul_rn(d_x, y), __dmul_rn(tp2, y)), __dmul_rn(tp1, x));
    const double fy_y = __dadd_rn(__dadd_rn(__dadd_rn(d, __dmul_rn(d_y, y)), __dmul_rn(tp2, x)), __dmul_rn(sp1, y));
    const double den = __dsub_rn(__dmul_rn(fy_x, fx_y), __dmul_rn(fx_x, fy_y));
    if (fabs(den) > 1e-3) {
      x = __dadd_rn(x, __ddiv_rn(__dsub_rn(__dmul_rn(fx, fy_y), __dmul_rn(fy, fx_y)), den));
      y = __dadd_rn(y, __ddiv_rn(__dsub_rn(__dmul_rn(fy, fx_x), __dmul_rn(fx, fy_x)), den));
    }
  }
  u = __double2float_rn(x);
  v = __double2float_rn(y);
}

// [NS] Cameras._generate_rays_from_coords: camera-space direction (OpenGL axes) of normalised image coordinates (u, v)
__device__ __forceinline__ void camera_direction(int camera_type, float u, float v, float d[3]) {
  if (camera_type == FNR_CAMERA_FISHEYE) {
    // theta = clip(|(u, v)|, 0, pi); (u sin(theta) / theta, v sin(theta) / theta, -cos(theta)).  At theta = 0 the reference
    // divides 0 by 0; that pixel is the optical axis (0, 0, -1) here.
    const float theta = fminf(sqrtf(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v))), CUDART_PI_F);
    float s, c;
    sincosf(theta, &s, &c);
    const float k = theta > 0.f ? __fdiv_rn(s, theta) : 0.f;
    d[0] = __fmul_rn(u, k);
    d[1] = __fmul_rn(v, k);
    d[2] = -c;
  } else if (camera_type == FNR_CAMERA_EQUIRECTANGULAR) {
    // theta = -pi u (azimuth), phi = pi (0.5 - v) (polar angle from +y)
    const float theta = __fmul_rn(-CUDART_PI_F, u), phi = __fmul_rn(CUDART_PI_F, __fsub_rn(0.5f, v));
    float st, ct, sp, cp;
    sincosf(theta, &st, &ct);
    sincosf(phi, &sp, &cp);
    d[0] = -__fmul_rn(st, sp);
    d[1] = cp;
    d[2] = -__fmul_rn(ct, sp);
  } else {
    d[0] = u;
    d[1] = v;
    d[2] = -1.0f;
  }
}

// The lens branch: pixel (x, y) of a camera with fp32 intrinsics and an optional [6] distortion -> camera-space direction.
// The pixel step divides with __fdiv_rn, as the pinhole training rays do; equirectangular cameras are not undistorted.
__device__ __forceinline__ void lens_direction(int x, int y, float fx, float fy, float cx, float cy, const float* __restrict__ dist,
                                               int camera_type, float d[3]) {
  float u = __fdiv_rn(__fsub_rn(__fadd_rn((float)x, 0.5f), cx), fx);
  float v = -__fdiv_rn(__fsub_rn(__fadd_rn((float)y, 0.5f), cy), fy);
  if (dist && camera_type != FNR_CAMERA_EQUIRECTANGULAR) undistort_rt(dist, u, v);
  camera_direction(camera_type, u, v, d);
}

// origin and d = normalize(R d_cam) of a [3][4] row-major c2w: rounded products, 3-term sums left to right (the training rays)
__device__ __forceinline__ void world_ray(const float* __restrict__ m, const float d[3], float* __restrict__ origin, float* __restrict__ dir) {
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = __fadd_rn(__fadd_rn(__fmul_rn(m[4 * k], d[0]), __fmul_rn(m[4 * k + 1], d[1])), __fmul_rn(m[4 * k + 2], d[2]));
  const float n = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(w[0], w[0]), __fmul_rn(w[1], w[1])), __fmul_rn(w[2], w[2]))), 1e-12f);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    origin[k] = m[4 * k + 3];
    dir[k] = __fdiv_rn(w[k], n);
  }
}

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
