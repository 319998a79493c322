// Kernels of the FruitNeRF hot path: one thread per sample point, per-ray compositing by one warp per ray.
//
// The field kernels (forward, export, backward) are instantiated per family C (CfgSmall, CfgBig) and implementation TC,
// and evaluate their Linear layers through a layer type (FieldLayers) that names each layer by its Slot.  TC = false is
// the "simt" implementation on Layers<C, false>, the exact-fp32 device path: MLP weights read straight from the torch
// parameter tensors through the read-only path (warp-uniform addresses, float4 where the row alignment allows); it is the
// on-device fp32 reference the tensor-core path is checked against at full size.  TC = true runs the MLP layers
// warpgroup-wide on the Hopper tensor cores (fnr_wgmma.cuh): the big family on Layers<CfgBig, true>, which stages each
// layer's weights at every step, the small family on ResidentLayers<Plan>, persistent CTAs that hold the weights in
// shared memory.  The layer type also gives its kernels' launch geometry.
//
// Reference semantics: fruit_nerf/fruit_field.py:168-301, fruit_nerf/fruit_nerf.py:251-269,316-357.
#include <type_traits>
#include "fnr_common.cuh"
#include "fnr_kernels.h"
#include "fnr_wgmma.cuh"

namespace fnr {

constexpr int kThreads = 128;

// The field's Linear layers.  The first six are the small family's tensor-core layers in the order of its resident
// weight image; kSem2 exists in the big family only.
enum Slot { kBase0, kBase1, kSem0, kSem1, kCol0, kCol1, kHead, kCol2, kSem2 };

template <int GEO_, int SEM_LAYERS_, int SEM_H_>
struct Cfg {
  static constexpr int L = 16, ENC = 32;
  static constexpr int GEO = GEO_;
  static constexpr int BASE_H = 64, BASE_OUT = 1 + GEO_;
  static constexpr int SEM_LAYERS = SEM_LAYERS_;  // Linear layers inside mlp_semantics
  static constexpr int SEM_H = SEM_H_, SEM_OUT = 64;
  static constexpr int APP = 32, SH = 16;
  static constexpr int COL_IN = SH + GEO_ + APP, COL_H = 64;
  static constexpr int MAXW = (SEM_H_ > COL_IN ? SEM_H_ : COL_IN) > 64 ? (SEM_H_ > COL_IN ? SEM_H_ : COL_IN) : 64;
  // Shape of slot s's layer W [N][K]; 0 for a slot the family does not have
  static constexpr int K(int s) {
    return s == kBase0 ? ENC : s == kBase1 ? BASE_H : s == kSem0 ? GEO : s == kSem1 ? SEM_H : s == kSem2 ? (SEM_LAYERS == 3 ? SEM_H : 0)
         : s == kCol0 ? COL_IN : s == kHead ? SEM_OUT : COL_H;
  }
  static constexpr int N(int s) {
    return s == kBase0 ? BASE_H : s == kBase1 ? BASE_OUT : s == kSem0 ? SEM_H : s == kSem1 ? (SEM_LAYERS == 3 ? SEM_H : SEM_OUT)
         : s == kSem2 ? (SEM_LAYERS == 3 ? SEM_OUT : 0) : s == kHead ? 1 : s == kCol2 ? 3 : COL_H;
  }
};
using CfgSmall = Cfg<15, 2, 64>;
using CfgBig = Cfg<30, 3, 128>;

// ------------------------------------------------------------------------------------------
// Dense layers on per-thread register vectors.  Weight rows are warp-uniform global addresses.
// A = alignment (in floats, 0..3) of the row start relative to a 16-byte boundary.
// ------------------------------------------------------------------------------------------
template <int K, int A>
__device__ __forceinline__ float dot_row(const float* __restrict__ w, const float (&x)[K], float acc) {
  constexpr int HEAD = ((4 - A) & 3) < K ? ((4 - A) & 3) : K;
  constexpr int BODY = (K - HEAD) / 4;
#pragma unroll
  for (int k = 0; k < HEAD; ++k) acc = fmaf(__ldg(w + k), x[k], acc);
#pragma unroll
  for (int i = 0; i < BODY; ++i) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(w + HEAD + 4 * i));
    acc = fmaf(v.x, x[HEAD + 4 * i + 0], acc);
    acc = fmaf(v.y, x[HEAD + 4 * i + 1], acc);
    acc = fmaf(v.z, x[HEAD + 4 * i + 2], acc);
    acc = fmaf(v.w, x[HEAD + 4 * i + 3], acc);
  }
#pragma unroll
  for (int k = HEAD + 4 * BODY; k < K; ++k) acc = fmaf(__ldg(w + k), x[k], acc);
  return acc;
}

template <int K, int A>
__device__ __forceinline__ void axpy_row(const float* __restrict__ w, float g, float (&dx)[K]) {
  constexpr int HEAD = ((4 - A) & 3) < K ? ((4 - A) & 3) : K;
  constexpr int BODY = (K - HEAD) / 4;
#pragma unroll
  for (int k = 0; k < HEAD; ++k) dx[k] = fmaf(__ldg(w + k), g, dx[k]);
#pragma unroll
  for (int i = 0; i < BODY; ++i) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(w + HEAD + 4 * i));
    dx[HEAD + 4 * i + 0] = fmaf(v.x, g, dx[HEAD + 4 * i + 0]);
    dx[HEAD + 4 * i + 1] = fmaf(v.y, g, dx[HEAD + 4 * i + 1]);
    dx[HEAD + 4 * i + 2] = fmaf(v.z, g, dx[HEAD + 4 * i + 2]);
    dx[HEAD + 4 * i + 3] = fmaf(v.w, g, dx[HEAD + 4 * i + 3]);
  }
#pragma unroll
  for (int k = HEAD + 4 * BODY; k < K; ++k) dx[k] = fmaf(__ldg(w + k), g, dx[k]);
}

// y = act(W x + b),  W [N][K] row-major (16-byte aligned base).
template <int K, int N, bool RELU>
__device__ __forceinline__ void linear_fwd(const float* __restrict__ W, const float* __restrict__ b, const float (&x)[K],
                                           float (&y)[N]) {
  constexpr int N4 = N / 4 * 4;
  for (int n = 0; n < N4; n += 4) {
    const float* w = W + (size_t)n * K;
    float a0 = dot_row<K, 0>(w, x, __ldg(b + n));
    float a1 = dot_row<K, (K) & 3>(w + K, x, __ldg(b + n + 1));
    float a2 = dot_row<K, (2 * K) & 3>(w + 2 * K, x, __ldg(b + n + 2));
    float a3 = dot_row<K, (3 * K) & 3>(w + 3 * K, x, __ldg(b + n + 3));
    y[n] = RELU ? fmaxf(a0, 0.f) : a0;
    y[n + 1] = RELU ? fmaxf(a1, 0.f) : a1;
    y[n + 2] = RELU ? fmaxf(a2, 0.f) : a2;
    y[n + 3] = RELU ? fmaxf(a3, 0.f) : a3;
  }
  if (N - N4 >= 1) {
    float a = dot_row<K, 0>(W + (size_t)N4 * K, x, __ldg(b + N4));
    y[N4] = RELU ? fmaxf(a, 0.f) : a;
  }
  if (N - N4 >= 2) {
    float a = dot_row<K, (K) & 3>(W + (size_t)(N4 + 1) * K, x, __ldg(b + N4 + 1));
    y[N4 + 1 < N ? N4 + 1 : 0] = RELU ? fmaxf(a, 0.f) : a;
  }
  if (N - N4 >= 3) {
    float a = dot_row<K, (2 * K) & 3>(W + (size_t)(N4 + 2) * K, x, __ldg(b + N4 + 2));
    y[N4 + 2 < N ? N4 + 2 : 0] = RELU ? fmaxf(a, 0.f) : a;
  }
}

// dx = W^T dy
template <int K, int N>
__device__ __forceinline__ void linear_bwd_input(const float* __restrict__ W, const float (&dy)[N], float (&dx)[K]) {
#pragma unroll
  for (int k = 0; k < K; ++k) dx[k] = 0.f;
  constexpr int N4 = N / 4 * 4;
  for (int n = 0; n < N4; n += 4) {
    const float* w = W + (size_t)n * K;
    axpy_row<K, 0>(w, dy[n], dx);
    axpy_row<K, (K) & 3>(w + K, dy[n + 1], dx);
    axpy_row<K, (2 * K) & 3>(w + 2 * K, dy[n + 2], dx);
    axpy_row<K, (3 * K) & 3>(w + 3 * K, dy[n + 3], dx);
  }
  if (N - N4 >= 1) axpy_row<K, 0>(W + (size_t)N4 * K, dy[N4], dx);
  if (N - N4 >= 2) axpy_row<K, (K) & 3>(W + (size_t)(N4 + 1) * K, dy[N4 + 1 < N ? N4 + 1 : 0], dx);
  if (N - N4 >= 3) axpy_row<K, (2 * K) & 3>(W + (size_t)(N4 + 2) * K, dy[N4 + 2 < N ? N4 + 2 : 0], dx);
}

// ------------------------------------------------------------------------------------------
// Hash-grid encode of one point (fp32 table, float2 rows).
// ------------------------------------------------------------------------------------------
template <int L>
__device__ __forceinline__ void hash_encode(const float2* __restrict__ table, const float* __restrict__ scalings,
                                            uint32_t log2T, const Vec3& p, float (&enc)[2 * L]) {
#pragma unroll 2
  for (int l = 0; l < L; ++l) {
    const float2 r = level_gather(table, p, scalings[l], l, log2T);
    enc[2 * l] = r.x;
    enc[2 * l + 1] = r.y;
  }
}

// ------------------------------------------------------------------------------------------
// Field evaluation of one point.
// ------------------------------------------------------------------------------------------
// fp32 weight gradient of one layer over the CTA's 128-point tile (K4 below)
template <int K, int N>
__device__ __forceinline__ void tile_weight_grad(float* __restrict__ sX, float* __restrict__ sY, const float (&x)[K],
                                                 const float (&dy)[N], float* __restrict__ gW, float* __restrict__ gb);

constexpr int cmax(int a, int b) { return a > b ? a : b; }

// Slot s's weight W [N][K] and bias [N] in a parameter set: the parameters P, or the gradients G they are added into
__device__ __forceinline__ float* weight(const KParams& P, int s) {
  return s == kBase0 ? P.base_w[0] : s == kBase1 ? P.base_w[1] : s == kSem0 ? P.sem_w[0] : s == kSem1 ? P.sem_w[1] : s == kSem2 ? P.sem_w[2]
       : s == kCol0 ? P.col_w[0] : s == kCol1 ? P.col_w[1] : s == kHead ? P.head_w : P.col_w[2];
}
__device__ __forceinline__ float* bias(const KParams& P, int s) {
  return s == kBase0 ? P.base_b[0] : s == kBase1 ? P.base_b[1] : s == kSem0 ? P.sem_b[0] : s == kSem1 ? P.sem_b[1] : s == kSem2 ? P.sem_b[2]
       : s == kCol0 ? P.col_b[0] : s == kCol1 ? P.col_b[1] : s == kHead ? P.head_b : P.col_b[2];
}

// The field kernels evaluate their Linear layers through a layer type (Layers<C, TC> or ResidentLayers<Plan>).  Both
// have the same calls, each naming its layer by SLOT, whose shape the register arrays must have:
//   fwd<SLOT, RELU>(P, x, y)           y = act(W x + b)
//   fwd2<S0, S1, RELU1>(P, x, m, y)    m = relu(W0 x + b0), y = act(W1 m + b1)
//   dx<SLOT>(P, dy, dxv)               dxv = W^T dy
//   dw<SLOT>(G, x, dy)                 dW = dY^T X and db over the warpgroup's 128-point tile, added to G
//   grad<SLOT>(P, G, x, dy, dxv)       dx and dw
//   grad_relu<SLOT>(P, G, x, dy, dxv)  grad of a layer whose input x is a ReLU's output, dxv masked by that ReLU (x > 0)
// and the same launch geometry of their kernels:
//   kGroups                            MMA warpgroups per CTA (each takes its own 128-point tiles)
//   kThreadsPerCta, kMinCtas           the kernels' __launch_bounds__ (kMinCtas = 0: none given)
//   kFwdSmemBytes, kBwdSmemBytes       dynamic shared memory of the forward and export, and of the backward
//   kResident                          one persistent CTA per SM on the resident weight image (the small family's
//                                      tensor-core kernels); otherwise as many CTAs as fit on the SMs
// Layers<C, TC> evaluates a layer in CTAs of one warpgroup.  TC = false: per thread in fp32 on the CUDA cores (the exact
// device reference).  TC = true: warpgroup-wide on the tensor cores with the weight tile staged from global memory at
// every step (fnr_wgmma.cuh; every thread of the 128-thread CTA must take part): the big family's tensor-core path.
template <class C, bool TC>
struct Layers {
  static constexpr int kGroups = 1;
  static constexpr int kThreadsPerCta = kThreads;
  static constexpr int kMinCtas = 0;
  static constexpr bool kResident = false;
  // the 1- and 3-wide output heads (64 MACs per point) stay in exact fp32 on the CUDA cores on both paths
  static constexpr bool tensor(int n) { return TC && n >= 8; }
  // dynamic shared memory: the sX / sY tiles of tile_weight_grad, and the wgmma operand plans (the backward's heads
  // still use tile_weight_grad, so its tensor-core plan holds that tile too)
  static constexpr int kTileFloats = ((C::MAXW + 3) & ~3) + 4;  // padded row stride of sX / sY
  static constexpr int kTileBytes = 2 * kThreads * kTileFloats * 4;
  static constexpr int kFwdSmemBytes = TC ? wg::Smem<C::MAXW, C::MAXW>::kBytes : 0;
  static constexpr int kBwdSmemBytes =
      TC ? cmax(cmax(wg::Smem<C::MAXW, C::MAXW>::kBytes, wg::DwSmem<C::MAXW, C::MAXW>::kBytes), kTileBytes) : kTileBytes;

  static __device__ __forceinline__ uint8_t* dyn_smem() {
    extern __shared__ __align__(128) uint8_t wg_smem[];
    return wg_smem;
  }
  static __device__ __forceinline__ float* sX() { return reinterpret_cast<float*>(dyn_smem()); }
  static __device__ __forceinline__ float* sY() { return sX() + kThreads * kTileFloats; }

  // The layer arithmetic on the slot's pointers.  Each call below reads all of its pointers before any arithmetic (fwd2:
  // both layers'), where the call sites read them when they passed the pointers.  This is a codegen guard, not a
  // semantic requirement: the position of the parameter loads steers ptxas's register allocation, and reading them
  // later changed the SASS of the backward kernels.
  template <bool RELU, int Kv, int Nv>
  static __device__ __forceinline__ void linear(const float* __restrict__ W, const float* __restrict__ b, const float (&x)[Kv],
                                                float (&y)[Nv]) {
    if constexpr (tensor(Nv))
      wg::linear<C::MAXW, C::MAXW, Kv, Nv, RELU>(dyn_smem(), W, b, x, y);
    else
      linear_fwd<Kv, Nv, RELU>(W, b, x, y);
  }
  template <int Kv, int Nv>
  static __device__ __forceinline__ void input_grad(const float* __restrict__ W, const float (&dy)[Nv], float (&dxv)[Kv]) {
    if constexpr (tensor(Nv))
      wg::linear_dx<C::MAXW, C::MAXW, Kv, Nv>(dyn_smem(), W, dy, dxv);
    else
      linear_bwd_input<Kv, Nv>(W, dy, dxv);
    FNR_PHASE(kPhDx);
  }
  template <int Kv, int Nv>
  static __device__ __forceinline__ void weight_grad(const float (&x)[Kv], const float (&dy)[Nv], float* gW, float* gb) {
    if constexpr (tensor(Nv))
      wg::weight_grad<Kv, Nv>(dyn_smem(), x, dy, gW, gb);
    else
      tile_weight_grad<Kv, Nv>(sX(), sY(), x, dy, gW, gb);
    FNR_PHASE(kPhDw);
  }

  template <int SLOT, bool RELU, int Kv, int Nv>
  static __device__ __forceinline__ void fwd(const KParams& P, const float (&x)[Kv], float (&y)[Nv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv, "slot shape");
    linear<RELU>(weight(P, SLOT), bias(P, SLOT), x, y);
  }
  // two steps
  template <int S0, int S1, bool RELU1, int K0, int N0, int N1>
  static __device__ __forceinline__ void fwd2(const KParams& P, const float (&x)[K0], float (&m)[N0], float (&y)[N1]) {
    static_assert(C::K(S0) == K0 && C::N(S0) == N0 && C::K(S1) == N0 && C::N(S1) == N1, "slot shapes");
    const float *W0 = weight(P, S0), *b0 = bias(P, S0), *W1 = weight(P, S1), *b1 = bias(P, S1);
    linear<true>(W0, b0, x, m);
    linear<RELU1>(W1, b1, m, y);
  }
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void dx(const KParams& P, const float (&dy)[Nv], float (&dxv)[Kv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv, "slot shape");
    input_grad(weight(P, SLOT), dy, dxv);
  }
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void dw(const KParams& G, const float (&x)[Kv], const float (&dy)[Nv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv, "slot shape");
    weight_grad(x, dy, weight(G, SLOT), bias(G, SLOT));
  }
  // dx, then dw
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void grad(const KParams& P, const KParams& G, const float (&x)[Kv], const float (&dy)[Nv],
                                              float (&dxv)[Kv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv, "slot shape");
    const float* W = weight(P, SLOT);
    float *gW = weight(G, SLOT), *gb = bias(G, SLOT);
    input_grad(W, dy, dxv);
    weight_grad(x, dy, gW, gb);
  }
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void grad_relu(const KParams& P, const KParams& G, const float (&x)[Kv], const float (&dy)[Nv],
                                                   float (&dxv)[Kv]) {
    grad<SLOT>(P, G, x, dy, dxv);
#pragma unroll
    for (int k = 0; k < Kv; ++k) dxv[k] = x[k] > 0.f ? dxv[k] : 0.f;
  }
};

// The small family's tensor-core kernels (forward, export, backward) run persistent CTAs of G warpgroups, each warpgroup
// taking its own 128-point tiles.  Per CTA, the six tensor-core layers are split once into a resident bf16 hi / lo image
// (the K-major tiles rowgemm stages, so every layer runs the staged path's bytes and MMA sequence; dx reads the same image
// MN-major).  The backward also accumulates the weight gradients of all eight layers in fp32 in shared memory and adds
// them to the global gradient once, when the CTA ends.
// The resident plan of the small family: shape of every slot, offsets of its weight image (six tensor-core layers) and of
// its fp32 gradient accumulator (all eight; wg::DwAcc layout for the tensor-core layers, [N][K] then [N] for the heads).
namespace resident {
using C = CfgSmall;
static_assert(C::SEM_LAYERS == 2, "resident plan of the two-layer semantic MLP");
constexpr int kSlots = 8;  // kBase0 .. kCol2
constexpr int kImageSlots = 6;
constexpr bool tensor(int n) { return n >= 8; }
constexpr int img_bytes(int s) { return 2 * wg::padn(C::N(s)) * wg::pad16(C::K(s)) * 2; }
constexpr int img_off(int s) { return s == 0 ? 0 : img_off(s - 1) + img_bytes(s - 1); }
constexpr int kImageBytes = img_off(kImageSlots);
static_assert(kImageBytes == 64 * 1024, "16384 split weights");
constexpr int acc_floats(int s) {
  return tensor(C::N(s)) ? (C::N(s) + 15) / 16 * 32 * (wg::padn(C::K(s)) / 2) + C::N(s) : C::N(s) * C::K(s) + C::N(s);
}
constexpr int acc_off(int s) { return s == 0 ? 0 : acc_off(s - 1) + (acc_floats(s - 1) + 3) / 4 * 4; }  // float4-aligned
constexpr int align128(int b) { return (b + 127) / 128 * 128; }
}  // namespace resident

// The resident forward and export CTA: kGroups MMA warpgroups and one gather warpgroup (warpgroup kGroups).  The gather
// warpgroup gathers the last kGatherLevels levels of the hash grid for the MMA warpgroups' points and hands them over
// through a ring of kRing slots, each with a full and an empty mbarrier; the MMA warpgroups gather the other levels
// themselves.  Registers: launched at 168 per thread (384 threads, 64 512 of the SM's 65 536), the gather warpgroup drops
// to kGatherRegs and the MMA warpgroups rise to kMmaRegs.  The ring is kept small because the gather runs out of L1,
// which gets what shared memory leaves: a 64 KiB cp.async stage and a ring of four slots were measured slower, as was
// the gather warpgroup taking more than half of the levels (DESIGN.md section 4.3).
// Dynamic shared memory: weight image | per-warpgroup step tiles | ring slots | ring barriers.
struct ForwardPlan {
  static constexpr int kGroups = 2;
  static constexpr int kThreadsPerCta = (kGroups + 1) * kThreads;
  // one CTA per SM named in __launch_bounds__, so that ptxas knows the registers at entry (168) and can apply setmaxnreg
  static constexpr int kMinCtas = 1;
  static constexpr int kGatherRegs = 56, kMmaRegs = 224;
  static_assert(kThreads * (kGatherRegs + kGroups * kMmaRegs) <= kThreadsPerCta * 168, "register split of the CTA");
  static constexpr int kGatherLevels = 8;
  static constexpr int kRing = 2;
  static constexpr int kSlotFloats = kThreads * 2 * kGatherLevels;  // fp32, element (row, c) at (c / 4) * 512 + row * 4 + c % 4
  static constexpr int kStepOff = resident::kImageBytes;
  static constexpr int kRingOff = kStepOff + kGroups * wg::kResidentStepBytes;
  static constexpr int kBarOff = kRingOff + kRing * kSlotFloats * 4;
  static constexpr int kBytes = kBarOff + 2 * kRing * 8;
  // with the kernels' static shared memory (s_app, 128 B), within the 232 448 bytes an H100 CTA can have
  static_assert(kBytes + 128 <= 232448, "forward shared-memory plan");
};
// Dynamic shared memory of the resident backward CTA: weight image | accumulators | locks | per-warpgroup step tiles |
// per-warpgroup dW operand regions.
struct BackwardPlan {
  static constexpr int kGroups = 2;
  static constexpr int kThreadsPerCta = kGroups * kThreads;
  static constexpr int kMinCtas = 0;
  static constexpr int kAccOff = resident::kImageBytes;
  static constexpr int kLockOff = kAccOff + resident::acc_off(resident::kSlots) * 4;
  static constexpr int kStepOff = resident::align128(kLockOff + resident::kSlots * 4);
  static constexpr int kDwOff = kStepOff + kGroups * wg::kResidentStepBytes;
  static constexpr int kBytes = kDwOff + kGroups * wg::kDwXBytes;
  // with the kernel's static shared memory (s_app, 128 B; the phase timers' 112 B in that diagnostic build), within the
  // 232 448 bytes an H100 CTA can have
  static_assert(kBytes + 256 <= 232448, "backward shared-memory plan");
};

// The layers of the small family's tensor-core kernels on the resident image (Plan: the kernel's shared-memory plan).
// fwd and fwd2 are the same code in the forward, the export and the backward's recompute; acc / lock / part, prepare, flush, dx
// and dw exist in the backward's plan only.  One plan per kernel, so both shared-memory sizes are the plan's.
template <class Plan>
struct ResidentLayers {
  using C = CfgSmall;
  static constexpr int kGroups = Plan::kGroups;
  static constexpr int kThreadsPerCta = Plan::kThreadsPerCta;
  static constexpr int kMinCtas = Plan::kMinCtas;
  static constexpr int kFwdSmemBytes = Plan::kBytes, kBwdSmemBytes = Plan::kBytes;
  static constexpr bool kResident = true;
  static constexpr int kSlots = resident::kSlots;
  static constexpr bool tensor(int n) { return resident::tensor(n); }
  static constexpr int img_off(int s) { return resident::img_off(s); }
  static constexpr int acc_off(int s) { return resident::acc_off(s); }

  static __device__ __forceinline__ uint8_t* smem() {
    extern __shared__ __align__(128) uint8_t wg_smem[];
    return wg_smem;
  }
  static __device__ __forceinline__ uint8_t* step() { return smem() + Plan::kStepOff + wg::group() * wg::kResidentStepBytes; }
  static __device__ __forceinline__ uint8_t* dw_region() { return smem() + Plan::kDwOff + wg::group() * wg::kDwXBytes; }
  template <int S>
  static __device__ __forceinline__ float* acc() {
    constexpr int off = acc_off(S);
    return reinterpret_cast<float*>(smem() + Plan::kAccOff) + off;
  }
  static __device__ __forceinline__ int* lock(int s) { return reinterpret_cast<int*>(smem() + Plan::kLockOff) + s; }

  // Split slot S's weights into the image exactly as rowgemm stages them (getw(n, k) = W[n][k], zero padding).
  template <int S>
  static __device__ __forceinline__ void split_image(const KParams& P) {
    constexpr int NP = wg::padn(C::N(S)), KP = wg::pad16(C::K(S)), kChunks = NP * KP / 8;
    const float* __restrict__ W = weight(P, S);
    uint8_t* hi = smem() + img_off(S);
    for (int i = threadIdx.x; i < kChunks; i += blockDim.x) {
      const int n = i % NP, kc = i / NP;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (n < C::N(S) && 8 * kc + j < C::K(S)) ? __ldg(W + (size_t)n * C::K(S) + 8 * kc + j) : 0.f;
      wg::split_store8(hi, hi + NP * KP * 2, kc * (NP * 16) + n * 16, v);
    }
  }
  static __device__ __forceinline__ void split_all(const KParams& P) {
    split_image<kBase0>(P);
    split_image<kBase1>(P);
    split_image<kSem0>(P);
    split_image<kSem1>(P);
    split_image<kCol0>(P);
    split_image<kCol1>(P);
  }
  // Once per CTA, before the first tile: the weight image and the ring's barriers (forward and export).
  static __device__ __forceinline__ void build_image(const KParams& P) {
    split_all(P);
    if (threadIdx.x < Plan::kRing) {
      wg::mbar_init(full(threadIdx.x), kThreads);
      wg::mbar_init(empty(threadIdx.x), kThreads);
    }
    wg::fence_proxy_async();
    __syncthreads();
  }
  // The forward's ring: slot s's encoding rows, and its full (the gather warpgroup's 128 threads arrive) and empty (the
  // MMA warpgroup's 128 threads arrive) barriers.
  static __device__ __forceinline__ float* slot(int s) { return reinterpret_cast<float*>(smem() + Plan::kRingOff) + s * Plan::kSlotFloats; }
  static __device__ __forceinline__ uint64_t* full(int s) { return reinterpret_cast<uint64_t*>(smem() + Plan::kBarOff) + s; }
  static __device__ __forceinline__ uint64_t* empty(int s) { return full(Plan::kRing) + s; }
  // The encoding rows of this MMA warpgroup's k-th tile: ring item k * kGroups + group, in slot item % kRing at the
  // slot's (item / kRing)-th use.  The slot is released as soon as the row is in registers.
  static __device__ __forceinline__ void ring_read(long long k, float (&enc)[C::ENC]) {
    const long long item = k * kGroups + wg::group();
    const int s = (int)(item % Plan::kRing);
    wg::mbar_wait(full(s), (uint32_t)(item / Plan::kRing) & 1u);
    const float* row = slot(s) + 4 * wg::tid();
    constexpr int e0 = 2 * (C::L - Plan::kGatherLevels);
#pragma unroll
    for (int i = 0; i < Plan::kGatherLevels / 2; ++i) {
      const float4 v = *reinterpret_cast<const float4*>(row + i * wg::kRowsGroupStride);
      enc[e0 + 4 * i] = v.x;
      enc[e0 + 4 * i + 1] = v.y;
      enc[e0 + 4 * i + 2] = v.z;
      enc[e0 + 4 * i + 3] = v.w;
    }
    wg::mbar_arrive(empty(s));
  }
  // Once per CTA, before the first tile: the weight image, zero accumulators and free locks (backward).
  static __device__ __forceinline__ void prepare(const KParams& P) {
    split_all(P);
    constexpr int kAccFloats = acc_off(kSlots);
    float* a = acc<0>();
    for (int i = threadIdx.x; i < kAccFloats; i += blockDim.x) a[i] = 0.f;
    if (threadIdx.x < kSlots) *lock(threadIdx.x) = 0;
    wg::fence_proxy_async();
    __syncthreads();
  }
  // Slot S's accumulator added to the global gradient (reds: G may be a buffer other GPUs add into); after a CTA barrier.
  template <int S>
  static __device__ __forceinline__ void flush(const KParams& G) {
    constexpr int Kv = C::K(S), Nv = C::N(S);
    float* gW = weight(G, S);
    float* gb = bias(G, S);
    const float* a = acc<S>();
    constexpr int kW = tensor(Nv) ? wg::DwAcc<Kv, Nv>::kW : Nv * Kv;
    for (int e = threadIdx.x; e < kW; e += blockDim.x) {
      int n = e / Kv, k = e % Kv;
      if constexpr (tensor(Nv)) wg::DwAcc<Kv, Nv>::at(e, n, k);
      const float v = a[e];
      if (n < Nv && k < Kv && v != 0.f) atomicAdd(gW + (size_t)n * Kv + k, v);
    }
    for (int n = threadIdx.x; n < Nv; n += blockDim.x)
      if (a[kW + n] != 0.f) atomicAdd(gb + n, a[kW + n]);
  }
  static __device__ __forceinline__ void flush_all(const KParams& G) {
    flush<kBase0>(G);
    flush<kBase1>(G);
    flush<kSem0>(G);
    flush<kSem1>(G);
    flush<kCol0>(G);
    flush<kCol1>(G);
    flush<kHead>(G);
    flush<kCol2>(G);
  }

  // The fp32 heads only: every tensor-core layer runs in a chained pair (fwd2).
  template <int SLOT, bool RELU, int Kv, int Nv>
  static __device__ __forceinline__ void fwd(const KParams& P, const float (&x)[Kv], float (&y)[Nv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv && !tensor(Nv), "slot shape");
    linear_fwd<Kv, Nv, RELU>(weight(P, SLOT), bias(P, SLOT), x, y);
  }
  // Two tensor-core layers chained (wg::resident_chain).  In the forward and the export, m goes from the first layer's
  // accumulators to the second layer's operand tile without a round trip through rows, and is left unset.  The backward,
  // whose weight gradients and ReLU masks read m, gets it as rows.  The bias and ReLU are the same fp32 operations either
  // way, so m and y have the same bits.
  template <int S0, int S1, bool RELU1, int K0, int N0, int N1>
  static __device__ __forceinline__ void fwd2(const KParams& P, const float (&x)[K0], float (&m)[N0], float (&y)[N1]) {
    static_assert(C::K(S0) == K0 && C::N(S0) == N0 && C::K(S1) == N0 && C::N(S1) == N1 && tensor(N0) && tensor(N1), "slot shapes");
    const float* __restrict__ b0 = bias(P, S0);
    const float* __restrict__ b1 = bias(P, S1);
    wg::resident_chain<wg::padn(N0), wg::pad16(K0), wg::padn(N1), std::is_same<Plan, BackwardPlan>::value>(
        step(), smem() + img_off(S0), smem() + img_off(S1), x, m, y, [&](int c, float v) { return fmaxf(v + __ldg(b0 + c), 0.f); });
#pragma unroll
    for (int n = 0; n < N1; ++n) {  // as wg::linear
      const float v = y[n] + __ldg(b1 + n);
      y[n] = RELU1 ? fmaxf(v, 0.f) : v;
    }
  }
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void dx(const KParams& P, const float (&dy)[Nv], float (&dxv)[Kv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv, "slot shape");
    if constexpr (tensor(Nv))
      wg::resident_rowgemm_t<wg::padn(Nv), wg::pad16(Kv)>(step(), smem() + img_off(SLOT), dy, dxv);
    else
      linear_bwd_input<Kv, Nv>(weight(P, SLOT), dy, dxv);
    FNR_PHASE(kPhDx);
  }
  // dW / db into the CTA's accumulators, which flush adds to G
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void dw(const KParams&, const float (&x)[Kv], const float (&dy)[Nv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv, "slot shape");
    if constexpr (tensor(Nv))
      wg::weight_grad_acc<Kv, Nv>(step(), dw_region(), x, dy, acc<SLOT>(), lock(SLOT));
    else
      wg::head_weight_grad_acc<Kv, Nv>(reinterpret_cast<float*>(dw_region()), x, dy, acc<SLOT>(), lock(SLOT));
    FNR_PHASE(kPhDw);
  }
  // Both gradients of one layer, the weight gradient first.  A tensor-core layer stages dy once: dW reads the tile
  // weight_grad_acc leaves in step(), and dx runs its MMAs on the same tile, so dy is dead once staged and not live next
  // to dxv (for a 64-wide layer, 64 registers at the backward's peak; DESIGN.md section 4.3).
  // RELU (grad_relu): x is a ReLU's output and dxv is masked by it.  Once dW has read x, only its signs are needed, so
  // they are kept as one bit per input (bit k % 32 of word k / 32) and the floats are dead before dx runs.
  // A head's W is read before dw runs, where the call sites read it when they passed it.  This is a codegen guard, not a
  // semantic requirement: reading it in dx moves the load and changes the backward kernel's register allocation; read
  // here, the kernel compiles to the SASS it had before the slot interface.
  template <int SLOT, bool RELU = false, int Kv, int Nv>
  static __device__ __forceinline__ void grad(const KParams& P, const KParams& G, const float (&x)[Kv], const float (&dy)[Nv],
                                              float (&dxv)[Kv]) {
    [[maybe_unused]] const float* W = weight(P, SLOT);
    dw<SLOT>(G, x, dy);
    uint32_t live[RELU ? (Kv + 31) / 32 : 1] = {};
    if constexpr (RELU) {
#pragma unroll
      for (int k = 0; k < Kv; ++k) live[k / 32] |= (x[k] > 0.f ? 1u : 0u) << (k % 32);
    }
    if constexpr (tensor(Nv))
      wg::resident_rowgemm_t_staged<wg::padn(Nv), wg::pad16(Kv), Nv>(step(), smem() + img_off(SLOT), dxv);
    else
      linear_bwd_input<Kv, Nv>(W, dy, dxv);
    FNR_PHASE(kPhDx);
    if constexpr (RELU) {
#pragma unroll
      for (int k = 0; k < Kv; ++k) dxv[k] = (live[k / 32] >> (k % 32)) & 1u ? dxv[k] : 0.f;
    }
  }
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void grad_relu(const KParams& P, const KParams& G, const float (&x)[Kv], const float (&dy)[Nv],
                                                   float (&dxv)[Kv]) {
    grad<SLOT, true>(P, G, x, dy, dxv);
  }
  // m = relu(W x + b) of a chained pair's first layer on its own, by the backward's row path of fwd2: the same tile
  // bytes, MMAs and fp32 bias and ReLU, so m has the bits fwd2 gives.  The backward recomputes the base MLP's h1 with it.
  template <int SLOT, int Kv, int Nv>
  static __device__ __forceinline__ void fwd_relu(const KParams& P, const float (&x)[Kv], float (&m)[Nv]) {
    static_assert(C::K(SLOT) == Kv && C::N(SLOT) == Nv && tensor(Nv), "slot shape");
    const float* __restrict__ b = bias(P, SLOT);
    wg::resident_rowgemm<wg::padn(Nv), wg::pad16(Kv)>(step(), smem() + img_off(SLOT), x, m);
#pragma unroll
    for (int n = 0; n < Nv; ++n) m[n] = fmaxf(m[n] + __ldg(b + n), 0.f);
  }
};
using ResidentForward = ResidentLayers<ForwardPlan>;

// The layers of family C's field kernels in implementation TC (Plan: ForwardPlan for the forward and the export,
// BackwardPlan for the backward): the small family's tensor-core kernels run on the resident image, the others on
// Layers<C, TC>.
template <class C, bool TC, class Plan>
using FieldLayers = std::conditional_t<TC && std::is_same<C, CfgSmall>::value, ResidentLayers<Plan>, Layers<C, TC>>;

template <class C>
struct Acts {
  float h1[C::BASE_H];      // relu(base0)
  float out[C::BASE_OUT];   // [h0, geo...]
  float z1[C::SEM_H];       // relu(sem0)
  float z2[C::SEM_LAYERS == 3 ? C::SEM_H : 1];  // relu(sem1) (3-layer variant)
  float zo[C::SEM_OUT];     // semantic MLP output (no activation)
  float cin[C::COL_IN];     // [sh16, geo, app]
  float c1[C::COL_H], c2[C::COL_H];
  float rgb[3];
  float logit;
};

// The field's branch forwards.  field_mlps and the backward's recompute both run these, so the recompute gives the
// forward's pre-activations bit for bit and its ReLU masks agree with the forward that ran.
//
// Lin: the layer type (FieldLayers).
//
// base MLP: enc -> [h0, geo...]; geo = out[1:]
template <class C, class Lin>
__device__ __forceinline__ void base_fwd(const KParams& P, const float (&enc)[C::ENC], float (&h1)[C::BASE_H],
                                         float (&out)[C::BASE_OUT], float (&geo)[C::GEO]) {
  Lin::template fwd2<kBase0, kBase1, false>(P, enc, h1, out);
#pragma unroll
  for (int i = 0; i < C::GEO; ++i) geo[i] = out[1 + i];
}

// semantic branch up to the logit head: mlp_semantics(detach(geo)) (fruit_field.py:263-268)
template <class C, class Lin>
__device__ __forceinline__ void semantic_fwd(const KParams& P, const float (&geo)[C::GEO], float (&z1)[C::SEM_H],
                                             float (&z2)[C::SEM_LAYERS == 3 ? C::SEM_H : 1], float (&zo)[C::SEM_OUT]) {
  if constexpr (C::SEM_LAYERS == 3) {
    Lin::template fwd<kSem0, true>(P, geo, z1);
    Lin::template fwd<kSem1, true>(P, z1, z2);
    Lin::template fwd<kSem2, false>(P, z2, zo);
  } else {
    Lin::template fwd2<kSem0, kSem1, false>(P, geo, z1, zo);
  }
}

// the colour MLP's input cat[SH(dir), geo, appearance]
template <class C>
__device__ __forceinline__ void colour_input(const float* __restrict__ dir, const float (&geo)[C::GEO], const float (&app)[C::APP],
                                             float (&cin)[C::COL_IN]) {
  sh_degree4(dir[0], dir[1], dir[2], cin);
#pragma unroll
  for (int i = 0; i < C::GEO; ++i) cin[C::SH + i] = geo[i];
#pragma unroll
  for (int i = 0; i < C::APP; ++i) cin[C::SH + C::GEO + i] = app[i];
}

// colour branch up to the sigmoid: cat[SH(dir), geo, appearance] -> MLP (fruit_field.py:270-278)
template <class C, class Lin>
__device__ __forceinline__ void colour_fwd(const KParams& P, const float* __restrict__ dir, const float (&geo)[C::GEO],
                                           const float (&app)[C::APP], float (&cin)[C::COL_IN], float (&c1)[C::COL_H],
                                           float (&c2)[C::COL_H], float (&o3)[3]) {
  colour_input<C>(dir, geo, app, cin);
  Lin::template fwd2<kCol0, kCol1, true>(P, cin, c1, c2);
  Lin::template fwd<kCol2, false>(P, c2, o3);
}

template <class C, class Lin>
__device__ __forceinline__ void field_mlps(const KParams& P, const float (&enc)[C::ENC], const float* __restrict__ dir,
                                           const float (&app)[C::APP], Acts<C>& a) {
  float geo[C::GEO];
  base_fwd<C, Lin>(P, enc, a.h1, a.out, geo);
  semantic_fwd<C, Lin>(P, geo, a.z1, a.z2, a.zo);
  float lg[1];
  Lin::template fwd<kHead, false>(P, a.zo, lg);
  a.logit = lg[0];
  float o3[3];
  colour_fwd<C, Lin>(P, dir, geo, app, a.cin, a.c1, a.c2, o3);
#pragma unroll
  for (int i = 0; i < 3; ++i) a.rgb[i] = sigmoidf_(o3[i]);
}

// The appearance vector of a point in the backward and export: its camera's embedding row (per-camera mode), else the
// block's s_app.
template <int APP>
__device__ __forceinline__ void load_appearance(const KParams& P, int mode, int cam, const float* s_app, float (&appv)[APP]) {
#pragma unroll
  for (int i = 0; i < APP; ++i) appv[i] = (mode == FNR_APP_PER_CAMERA) ? __ldg(P.app_embedding + (size_t)cam * APP + i) : s_app[i];
}

// Mean appearance embedding into shared memory (fruit_field.py:217-219, 254-256).
__device__ __forceinline__ void block_mean_embedding(const KParams& P, int num_images, int app_dim, int mode,
                                                     float* s_app) {
  if (threadIdx.x < app_dim) {
    float acc = 0.f;
    if (mode == FNR_APP_MEAN) {
      for (int i = 0; i < num_images; ++i) acc += __ldg(P.app_embedding + (size_t)i * app_dim + threadIdx.x);
      acc /= (float)num_images;
    }
    s_app[threadIdx.x] = acc;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------
// K1: per-point field forward.
// ------------------------------------------------------------------------------------------
// The small family's tensor-core forward and export run on the resident weight image (ResidentForward); the other
// instantiations stage the weights at every layer step (Layers<C, TC>) in CTAs of one warpgroup.
//
// The warpgroup of this thread in a CTA of G = Lin::kGroups MMA warpgroups, and the thread's index in it (G = 1: the
// CTA's own indices, so that the one-warpgroup kernels compile as they did before there were several)
template <int G>
__device__ __forceinline__ int group_of() { return G == 1 ? 0 : wg::group(); }
template <int G>
__device__ __forceinline__ unsigned thread_of() { return G == 1 ? threadIdx.x : (unsigned)wg::tid(); }

// The gather warpgroup of the resident forward and export.  It takes the tiles of the CTA's MMA warpgroups in the order
// they run them (ring item j: the (j / kGroups)-th tile of warpgroup j % kGroups), one point per thread, a point past N
// clamped to N - 1 as in the MMA warpgroups.  position(p) is the point's field_position.  Levels [L - kGatherLevels, L)
// go through level_gather, two per step as in hash_encode, so the encoding has its bits.  They go into ring slot
// j % kRing (and into the encoding stash, when there is one), and the slot's full barrier is arrived on.
template <class Position>
__device__ __forceinline__ void gather_encodings(const KField& F, const KParams& P, long long N, float* __restrict__ stash,
                                                 Position position) {
  using Plan = ForwardPlan;
  using RF = ResidentForward;
  constexpr int L = CfgSmall::L;
#ifdef FNR_FWD_NO_GATHER
  return;  // the MMA warpgroups make up their encodings (diagnostic build)
#endif
  const int t = wg::tid();
  const float2* __restrict__ table = reinterpret_cast<const float2*>(P.hash_table);
  for (long long j = 0;; ++j) {
    const long long tile = ((long long)blockIdx.x + j / Plan::kGroups * gridDim.x) * Plan::kGroups + j % Plan::kGroups;
    if (tile * kThreads >= N) break;
    const int s = (int)(j % Plan::kRing);
    const long long p = tile * kThreads + t;
    const bool valid = p < N;
    const Vec3 pos = position(valid ? p : N - 1);
    wg::mbar_wait(RF::empty(s), ((uint32_t)(j / Plan::kRing) & 1u) ^ 1u);  // the slot's previous row has been read
    float* row = RF::slot(s) + 4 * t;
#pragma unroll 1
    for (int cg = 0; cg < Plan::kGatherLevels / 2; ++cg) {  // column group of 4 floats = levels l0, l0 + 1
      const int l0 = L - Plan::kGatherLevels + 2 * cg;
      const float2 e0 = level_gather(table, pos, F.scalings[l0], l0, F.log2T);
      const float2 e1 = level_gather(table, pos, F.scalings[l0 + 1], l0 + 1, F.log2T);
      const float4 v = make_float4(e0.x, e0.y, e1.x, e1.y);
      *reinterpret_cast<float4*>(row + cg * wg::kRowsGroupStride) = v;
      if (stash && valid) reinterpret_cast<float4*>(stash + (size_t)p * CfgSmall::ENC)[l0 / 2] = v;
    }
    wg::mbar_arrive(RF::full(s));
  }
}

// The resident kernels' split of the CTA into the gather warpgroup, which runs gather_encodings and returns false, and
// the MMA warpgroups, which return true.
template <class Position>
__device__ __forceinline__ bool mma_warpgroup(const KField& F, const KParams& P, long long N, float* stash, Position position) {
  ResidentForward::build_image(P);
  if (wg::group() == ForwardPlan::kGroups) {
    wg::setmaxnreg_dec<ForwardPlan::kGatherRegs>();
    gather_encodings(F, P, N, stash, position);
    return false;
  }
  wg::setmaxnreg_inc<ForwardPlan::kMmaRegs>();
  return true;
}

// The encoding of an MMA warpgroup's k-th point: levels [0, L - kGatherLevels) gathered here with level_gather (four
// levels per step) and stored to the stash, when there is one; the others from the ring.  With
// -DFNR_FWD_NO_GATHER (a diagnostic build that times the MMA warpgroups alone) a made-up row.
__device__ __forceinline__ void resident_encoding(const KField& F, const KParams& P, long long k, const Vec3& pos, float* stash_row,
                                                  float (&enc)[CfgSmall::ENC]) {
#ifdef FNR_FWD_NO_GATHER
#pragma unroll
  for (int l = 0; l < CfgSmall::L; ++l) {
    enc[2 * l] = pos.x;
    enc[2 * l + 1] = pos.y + pos.z;
  }
#else
  constexpr int kOwn = CfgSmall::L - ForwardPlan::kGatherLevels;
  const float2* __restrict__ table = reinterpret_cast<const float2*>(P.hash_table);
#pragma unroll 2
  for (int cg = 0; cg < kOwn / 2; ++cg) {
    const float2 e0 = level_gather(table, pos, F.scalings[2 * cg], 2 * cg, F.log2T);
    const float2 e1 = level_gather(table, pos, F.scalings[2 * cg + 1], 2 * cg + 1, F.log2T);
    enc[4 * cg] = e0.x;
    enc[4 * cg + 1] = e0.y;
    enc[4 * cg + 2] = e1.x;
    enc[4 * cg + 3] = e1.y;
    if (stash_row) reinterpret_cast<float4*>(stash_row)[cg] = make_float4(e0.x, e0.y, e1.x, e1.y);
  }
  ResidentForward::ring_read(k, enc);
#endif
}

// Every warpgroup takes whole 128-point tiles, tile g of CTA b then every (gridDim.x * warpgroups)-th one after it; threads
// past N compute a clamped point and store nothing, so that the warpgroup-wide tensor-core layers see every thread.  A
// warpgroup syncs on its own barrier only (wg::sync): the tile loop has no CTA-wide barrier, and a warpgroup without
// tiles leaves at once.
template <class C, bool TC>
__global__ void __launch_bounds__(FieldLayers<C, TC, ForwardPlan>::kThreadsPerCta, FieldLayers<C, TC, ForwardPlan>::kMinCtas)
    simt_field_forward_kernel(KField F, KParams P, KRays Rr, KFieldOut O) {
  using Lin = FieldLayers<C, TC, ForwardPlan>;
  constexpr bool kResident = Lin::kResident;
  constexpr int kGroups = Lin::kGroups;
  __shared__ float s_app[C::APP];
  block_mean_embedding(P, F.num_images, C::APP, F.appearance_mode, s_app);
  const long long N = (long long)Rr.R * Rr.S;
  if constexpr (kResident) {
    const bool mma = mma_warpgroup(F, P, N, O.stash_encoding, [&](long long p) {
      const int r = (int)(p / Rr.S);
      bool sel;
      return field_position(Rr.origins + 3 * (size_t)r, Rr.directions + 3 * (size_t)r, Rr.starts[p], Rr.ends[p], F.position_mode,
                            F.aabb, sel);
    });
    if (!mma) return;
  }
  const int g = group_of<kGroups>();
  const unsigned t = thread_of<kGroups>();
  const unsigned span = kResident ? kGroups * kThreads : blockDim.x;  // points of a CTA's round of tiles
  long long k = 0;  // the warpgroup's tile count
  for (long long p0 = (long long)blockIdx.x * span + g * kThreads; p0 < N; p0 += (long long)gridDim.x * span, ++k) {
    const bool valid = p0 + t < N;
    const long long p = valid ? p0 + t : N - 1;
    const int r = (int)(p / Rr.S);
    const float* o = Rr.origins + 3 * (size_t)r;
    const float* d = Rr.directions + 3 * (size_t)r;
    bool sel;
    const Vec3 pos = field_position(o, d, Rr.starts[p], Rr.ends[p], F.position_mode, F.aabb, sel);
    float enc[C::ENC];
    if constexpr (kResident) {
      resident_encoding(F, P, k, pos, O.stash_encoding && valid ? O.stash_encoding + (size_t)p * C::ENC : nullptr, enc);
    } else {
      hash_encode<C::L>(reinterpret_cast<const float2*>(P.hash_table), F.scalings, F.log2T, pos, enc);
      if (O.stash_encoding && valid) {
        float4* st = reinterpret_cast<float4*>(O.stash_encoding + (size_t)p * C::ENC);
#pragma unroll
        for (int i = 0; i < C::ENC / 4; ++i) st[i] = make_float4(enc[4 * i], enc[4 * i + 1], enc[4 * i + 2], enc[4 * i + 3]);
      }
    }
    // not load_appearance: selecting the source row once compiles to ~130 fewer instructions in this kernel
    const float* app = (F.appearance_mode == FNR_APP_PER_CAMERA)
                           ? P.app_embedding + (size_t)Rr.camera_indices[r] * C::APP
                           : s_app;
    float appv[C::APP];
#pragma unroll
    for (int i = 0; i < C::APP; ++i) appv[i] = (F.appearance_mode == FNR_APP_PER_CAMERA) ? __ldg(app + i) : app[i];
    Acts<C> a;
    field_mlps<C, Lin>(P, enc, d, appv, a);
    if (!valid) continue;
    const float density = sel ? expf(a.out[0]) : 0.f;
    if (O.sample_density) O.sample_density[p] = density;
    if (O.sample_semantics) O.sample_semantics[p] = a.logit;
    if (O.sample_rgb) {
      O.sample_rgb[3 * p] = a.rgb[0];
      O.sample_rgb[3 * p + 1] = a.rgb[1];
      O.sample_rgb[3 * p + 2] = a.rgb[2];
    }
  }
}

// ------------------------------------------------------------------------------------------
// K2: per-ray compositing, one warp per ray (fruit_nerf.py:325-348).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) simt_composite_kernel(KRays Rr, KComposite Cm) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int S = Rr.S;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < Rr.R; r += gridDim.x * warps_per_block) {
    const size_t base = (size_t)r * S;
    float run_x = 0.f, run_w = 0.f;
    float acc = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, sem = 0.f;
    int median = S - 1;
    bool found = false;
    for (int c0 = 0; c0 < S; c0 += 32) {
      const int i = c0 + lane;
      const bool in = i < S;
      float x = 0.f;
      if (in) {
        const float delta = Rr.ends[base + i] - Rr.starts[base + i];
        x = delta * Cm.sample_density[base + i];
      }
      const float w = chunk_weight(x, in, lane, run_x);
      if (in) {
        if (Cm.weights) Cm.weights[base + i] = w;
        float c0r = Cm.sample_rgb[3 * (base + i)], c0g = Cm.sample_rgb[3 * (base + i) + 1], c0b = Cm.sample_rgb[3 * (base + i) + 2];
        if (Cm.clamp_rgb) {
          c0r = nan_to_num(c0r);
          c0g = nan_to_num(c0g);
          c0b = nan_to_num(c0b);
        }
        cr += w * c0r;
        cg += w * c0g;
        cb += w * c0b;
        sem += w * Cm.sample_semantics[base + i];
        acc += w;
      }
      if (!found) found = median_chunk(w, in, c0, lane, run_w, median);
    }
    acc = warp_sum(acc);
    cr = warp_sum(cr);
    cg = warp_sum(cg);
    cb = warp_sum(cb);
    sem = warp_sum(sem);
    if (lane == 0) {
      float lr = Cm.sample_rgb[3 * (base + S - 1)], lg = Cm.sample_rgb[3 * (base + S - 1) + 1], lb = Cm.sample_rgb[3 * (base + S - 1) + 2];
      if (Cm.clamp_rgb) {
        lr = nan_to_num(lr);
        lg = nan_to_num(lg);
        lb = nan_to_num(lb);
      }
      float orr = cr + lr * (1.0f - acc), og = cg + lg * (1.0f - acc), ob = cb + lb * (1.0f - acc);
      if (Cm.clamp_rgb) {
        orr = fminf(fmaxf(orr, 0.f), 1.f);
        og = fminf(fmaxf(og, 0.f), 1.f);
        ob = fminf(fmaxf(ob, 0.f), 1.f);
      }
      if (Cm.rgb) {
        Cm.rgb[3 * r] = orr;
        Cm.rgb[3 * r + 1] = og;
        Cm.rgb[3 * r + 2] = ob;
      }
      if (Cm.accumulation) Cm.accumulation[r] = acc;
      if (Cm.semantics) Cm.semantics[r] = sem;
      if (Cm.depth_index) Cm.depth_index[r] = median;
      if (Cm.depth) Cm.depth[r] = (Rr.starts[base + median] + Rr.ends[base + median]) / 2;
    }
  }
}

// ------------------------------------------------------------------------------------------
// K3: compositing backward, one warp per ray -> per-sample (d_density, d_rgb, d_logit).
//   w_i = (1 - e^{-x_i}) e^{-X_i},  X_i = sum_{j<i} x_j,  x = delta * sigma
//   dL/dx_j = G_j T_{j+1} - sum_{i>j} G_i w_i,   G_i = dL/dw_i
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) simt_composite_backward_kernel(KRays Rr, KCompositeBwd B) {
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  const int S = Rr.S;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < Rr.R; r += gridDim.x * warps_per_block) {
    const size_t base = (size_t)r * S;
    if (!B.weights) {  // field-only backward (FruitField.forward users): upstream is per-sample
      for (int i = lane; i < S; i += 32) {
        float* out = B.point_grads + 5 * (base + i);
        out[0] = B.d_sample_density ? B.d_sample_density[base + i] : 0.f;
        out[1] = B.d_sample_rgb ? B.d_sample_rgb[3 * (base + i)] : 0.f;
        out[2] = B.d_sample_rgb ? B.d_sample_rgb[3 * (base + i) + 1] : 0.f;
        out[3] = B.d_sample_rgb ? B.d_sample_rgb[3 * (base + i) + 2] : 0.f;
        out[4] = B.d_sample_semantics ? B.d_sample_semantics[base + i] : 0.f;
      }
      continue;
    }
    const float gr = B.d_rgb ? B.d_rgb[3 * r] : 0.f, gg = B.d_rgb ? B.d_rgb[3 * r + 1] : 0.f, gb = B.d_rgb ? B.d_rgb[3 * r + 2] : 0.f;
    const float gacc = B.d_accumulation ? B.d_accumulation[r] : 0.f;
    const float gsem = B.d_semantics ? B.d_semantics[r] : 0.f;
    const float acc = B.accumulation[r];
    const float lr = B.sample_rgb[3 * (base + S - 1)], lg = B.sample_rgb[3 * (base + S - 1) + 1], lb = B.sample_rgb[3 * (base + S - 1) + 2];
    // G_i = dL/dw_i of sample i < S (rgb = sum w c + (1 - acc) c_last)
    auto upstream = [&](int i) {
      float G = gr * (B.sample_rgb[3 * (base + i)] - lr) + gg * (B.sample_rgb[3 * (base + i) + 1] - lg) +
                gb * (B.sample_rgb[3 * (base + i) + 2] - lb) + gacc;
      if (B.d_weights) G += B.d_weights[base + i];
      if (B.pass_semantic_gradients) G += gsem * B.sample_semantics[base + i];
      return G;
    };
    // suffix sums sum_{k>i} G_k w_k: exact (chunk_suffix) for S <= 1024; longer rays keep "total - prefix"
    const bool exact_suffix = S <= 1024;
    float later_chunks = 0.f, tot = 0.f;
    if (exact_suffix) {
      later_chunks = later_chunks_sum(S, lane, [&](int i) { return upstream(i) * B.weights[base + i]; });
    } else {
      for (int i = lane; i < S; i += 32) tot += upstream(i) * B.weights[base + i];
      tot = warp_sum(tot);
    }
    float run_x = 0.f, run_gw = 0.f;
    for (int c0 = 0, ci = 0; c0 < S; c0 += 32, ++ci) {
      const int i = c0 + lane;
      const bool in = i < S;
      float x = 0.f, G = 0.f, w = 0.f, delta = 0.f;
      if (in) {
        delta = Rr.ends[base + i] - Rr.starts[base + i];
        x = delta * B.sample_density[base + i];
        w = B.weights[base + i];
        G = upstream(i);
      }
      const float xin = warp_incl_scan(x, lane);
      const float gw = G * w;
      float suffix;
      if (exact_suffix) {
        suffix = chunk_suffix(gw, later_chunks, ci, lane);
      } else {
        const float gwin = warp_incl_scan(gw, lane);
        suffix = tot - (run_gw + gwin);
        run_gw += __shfl_sync(kFull, gwin, 31);
      }
      if (in) {
        float dsig = weights_dsigma(delta, G, run_x, xin, suffix);
        if (B.d_sample_density) dsig += B.d_sample_density[base + i];
        float dr = w * gr, dg = w * gg, db = w * gb;
        if (i == S - 1) {
          dr += (1.0f - acc) * gr;
          dg += (1.0f - acc) * gg;
          db += (1.0f - acc) * gb;
        }
        if (B.d_sample_rgb) {
          dr += B.d_sample_rgb[3 * (base + i)];
          dg += B.d_sample_rgb[3 * (base + i) + 1];
          db += B.d_sample_rgb[3 * (base + i) + 2];
        }
        float dl = w * gsem;
        if (B.d_sample_semantics) dl += B.d_sample_semantics[base + i];
        float* out = B.point_grads + 5 * (base + i);
        out[0] = dsig;
        out[1] = dr;
        out[2] = dg;
        out[3] = db;
        out[4] = dl;
      }
      run_x += __shfl_sync(kFull, xin, 31);
    }
  }
}

// ------------------------------------------------------------------------------------------
// K4: per-point field backward.  Weight gradients: a warpgroup's 128 points form one tile; for every
// layer the tile's inputs X[128,K] and output grads dY[128,N] go to shared memory.  simt: each thread
// reduces a 4x4 block of dW = dY^T X over the tile, then adds it to the global gradient.  Tensor cores:
// the tile's dW is one MMA, added to the global gradient per tile (Layers<C, true>) or to accumulators in
// shared memory that the CTA flushes once (ResidentLayers<BackwardPlan>, small family).
// ------------------------------------------------------------------------------------------
template <int K, int N>
__device__ __forceinline__ void tile_weight_grad(float* __restrict__ sX, float* __restrict__ sY, const float (&x)[K],
                                                 const float (&dy)[N], float* __restrict__ gW, float* __restrict__ gb) {
  constexpr int KP = ((K + 3) & ~3) + 4, NP = ((N + 3) & ~3) + 4;  // padded row strides (floats)
  const int t = threadIdx.x;
  __syncthreads();  // previous users of sX/sY are done
#pragma unroll
  for (int k = 0; k < KP - 4; ++k) sX[t * KP + k] = k < K ? x[k < K ? k : 0] : 0.f;
#pragma unroll
  for (int n = 0; n < NP - 4; ++n) sY[t * NP + n] = n < N ? dy[n < N ? n : 0] : 0.f;
  __syncthreads();
  constexpr int KB = (K + 3) / 4, NB = (N + 3) / 4;
  for (int blk = t; blk < KB * NB; blk += kThreads) {
    const int kb = blk % KB, nb = blk / KB;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
    for (int p = 0; p < kThreads; ++p) {
      const float4 xv = *reinterpret_cast<const float4*>(sX + p * KP + 4 * kb);
      const float4 yv = *reinterpret_cast<const float4*>(sY + p * NP + 4 * nb);
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, ys[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ys[i], xs[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = 4 * nb + i, k = 4 * kb + j;
        if (n < N && k < K && acc[i][j] != 0.f) atomicAdd(gW + (size_t)n * K + k, acc[i][j]);
      }
  }
  // bias grads: column sums of dY
  for (int n = t; n < N; n += kThreads) {
    float s = 0.f;
    for (int p = 0; p < kThreads; ++p) s += sY[p * NP + n];
    if (s != 0.f) atomicAdd(gb + n, s);
  }
}

#ifdef FNR_BWD_PHASE_TIMERS
__device__ unsigned long long g_bwd_phase_cycles[kBwdPhases];
#endif

template <class C, bool TC>
__global__ void __launch_bounds__(FieldLayers<C, TC, BackwardPlan>::kThreadsPerCta, FieldLayers<C, TC, BackwardPlan>::kMinCtas)
    simt_field_backward_kernel(KField F, KParams P, KParams G, KRays Rr, KFieldBwd B) {
  using Lin = FieldLayers<C, TC, BackwardPlan>;
  constexpr bool kResident = Lin::kResident;
  constexpr int kGroups = Lin::kGroups;  // warpgroups (tiles in flight) per CTA
  __shared__ float s_app[C::APP];
  block_mean_embedding(P, F.num_images, C::APP, F.appearance_mode, s_app);
  if constexpr (kResident) Lin::prepare(P);
#ifdef FNR_BWD_PHASE_TIMERS
  if (threadIdx.x < 2 * kBwdPhases) phase::cycles[threadIdx.x / kBwdPhases][threadIdx.x % kBwdPhases] = 0;
  if (wg::tid() == 0) phase::last[wg::group()] = clock64();
  __syncthreads();
#endif
  const long long N = (long long)Rr.R * Rr.S;
  const long long tiles = (N + kThreads - 1) / kThreads;
  const int lane = threadIdx.x & 31;
  // warpgroup g of CTA b takes tiles b * kGroups + g, strided over all warpgroups of the grid
  for (long long tile = (long long)blockIdx.x * kGroups + wg::group(); tile < tiles; tile += (long long)gridDim.x * kGroups) {
    const long long p = tile * kThreads + wg::tid();
    const bool valid = p < N;
    const long long pc = valid ? p : N - 1;
    const int r = (int)(pc / Rr.S);
    const float* o = Rr.origins + 3 * (size_t)r;
    const float* d = Rr.directions + 3 * (size_t)r;
    bool sel;
    const Vec3 pos = field_position(o, d, Rr.starts[pc], Rr.ends[pc], F.position_mode, F.aabb, sel);
    float enc[C::ENC];
    // the point's encoding: the forward's stash, else gathered again at position() (the resident kernel loads it twice)
    auto load_encoding = [&](auto position) {
      if (B.stash_encoding) {
        const float4* st = reinterpret_cast<const float4*>(B.stash_encoding + (size_t)pc * C::ENC);
#pragma unroll
        for (int i = 0; i < C::ENC / 4; ++i) {
          const float4 v = st[i];
          enc[4 * i] = v.x;
          enc[4 * i + 1] = v.y;
          enc[4 * i + 2] = v.z;
          enc[4 * i + 3] = v.w;
        }
      } else {
        hash_encode<C::L>(reinterpret_cast<const float2*>(P.hash_table), F.scalings, F.log2T, position(), enc);
      }
    };
    load_encoding([&] { return pos; });
    const int cam = (F.appearance_mode == FNR_APP_PER_CAMERA) ? Rr.camera_indices[r] : 0;
    float appv[C::APP];
    if constexpr (!kResident) load_appearance(P, F.appearance_mode, cam, s_app, appv);
    // upstream per-point grads (zero for padding threads)
    const float* pg = B.point_grads + 5 * (size_t)pc;
    const float vm = valid ? 1.f : 0.f;
    const float d_sigma = pg[0] * vm;
    const float d_rgb[3] = {pg[1] * vm, pg[2] * vm, pg[3] * vm};
    const float d_logit = pg[4] * vm;
    FNR_PHASE(kPhLoad);

    // The forward is recomputed branch by branch with field_mlps' branch functions, and each branch is back-propagated
    // right after its forward: only the base MLP's activations live across the whole tile.  The resident kernel keeps
    // of them only geo and the density's gradient, and recomputes enc and h1 for the base backward (DESIGN.md section 4.3).
    float h1[C::BASE_H], out[C::BASE_OUT], geo[C::GEO];
    base_fwd<C, Lin>(P, enc, h1, out, geo);
    // trunc_exp backward: g * exp(clamp(x, -15, 15)); density = exp(h0) * selector
    auto density_grad = [&] { return sel ? d_sigma * expf(fminf(fmaxf(out[0], -15.f), 15.f)) : 0.f; };
    float dout0 = 0.f;
    if constexpr (kResident) dout0 = density_grad();
    FNR_PHASE(kPhRecompute);

    float d_geo[C::GEO];
#pragma unroll
    for (int i = 0; i < C::GEO; ++i) d_geo[i] = 0.f;

    // Warpgroup 1 of the resident kernel runs the colour branch first, so that the CTA's two warpgroups run different
    // layers rather than the same layers in step (DESIGN.md section 4.3); d_geo then adds the branches' terms in the
    // other order.  The resident kernel runs both iterations, the semantic branch in iteration `sem` and the colour
    // branch in the other, one copy of each in its code.  The other kernels run one iteration with both branches.
    const int sem = kResident ? wg::group() : 0;
#pragma unroll 1
    for (int br = 0; br < (kResident ? 2 : 1); ++br) {
      if (!kResident || br == sem) {
        // ---- semantic branch (its logit head is not needed: d_logit is the upstream gradient) ----------------------
        float z1[C::SEM_H], zo[C::SEM_OUT];
        float z2[C::SEM_LAYERS == 3 ? C::SEM_H : 1];
        semantic_fwd<C, Lin>(P, geo, z1, z2, zo);
        FNR_PHASE(kPhRecompute);
        float dlg[1] = {d_logit};
        float dzo[C::SEM_OUT];
        Lin::template grad<kHead>(P, G, zo, dlg, dzo);
        float dz1[C::SEM_H];
        if constexpr (C::SEM_LAYERS == 3) {
          float dz2[C::SEM_H];
          Lin::template grad_relu<kSem2>(P, G, z2, dzo, dz2);
          Lin::template grad_relu<kSem1>(P, G, z1, dz2, dz1);
        } else {
          Lin::template grad_relu<kSem1>(P, G, z1, dzo, dz1);
        }
        Lin::template dw<kSem0>(G, geo, dz1);
        if (F.pass_semantic_gradients) {
          float dg[C::GEO];
          Lin::template dx<kSem0>(P, dz1, dg);
#pragma unroll
          for (int i = 0; i < C::GEO; ++i) d_geo[i] += dg[i];
        }
      }
      if (!kResident || br != sem) {
        // ---- colour branch -------------------------------------------------------------------
        float cin[C::COL_IN], c1[C::COL_H], c2[C::COL_H], o3[3];
        // the resident kernel loads it here rather than with the point's inputs, so that it is not live through the base
        // and semantic branches (fewer spills, DESIGN.md section 4.3)
        if constexpr (kResident) load_appearance(P, F.appearance_mode, cam, s_app, appv);
        colour_fwd<C, Lin>(P, d, geo, appv, cin, c1, c2, o3);
        FNR_PHASE(kPhRecompute);
        float do3[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float rgb = sigmoidf_(o3[i]);
          do3[i] = d_rgb[i] * rgb * (1.0f - rgb);
        }
        float dc2[C::COL_H], dc1[C::COL_H], dcin[C::COL_IN];
        Lin::template grad_relu<kCol2>(P, G, c2, do3, dc2);
        Lin::template grad_relu<kCol1>(P, G, c1, dc2, dc1);
        if constexpr (kResident) {
          // cin again, from what built it, rather than carried through the col2 and col1 gradients
          load_appearance(P, F.appearance_mode, cam, s_app, appv);
          colour_input<C>(d, geo, appv, cin);
        }
        Lin::template grad<kCol0>(P, G, cin, dc1, dcin);
#pragma unroll
        for (int i = 0; i < C::GEO; ++i) d_geo[i] += dcin[C::SH + i];
        // appearance-embedding gradient (only the per-camera rows are parameters of the graph;
        // the mean embedding spreads 1/num_images to every row)
        if (F.appearance_mode == FNR_APP_PER_CAMERA) {
          const bool uniform = __all_sync(kFull, cam == __shfl_sync(kFull, cam, 0));
          if (uniform) {
#pragma unroll
            for (int i = 0; i < C::APP; ++i) {
              const float s = warp_sum(dcin[C::SH + C::GEO + i]);
              if (lane == 0 && s != 0.f) atomicAdd(G.app_embedding + (size_t)cam * C::APP + i, s);
            }
          } else {
#pragma unroll
            for (int i = 0; i < C::APP; ++i)
              if (dcin[C::SH + C::GEO + i] != 0.f) atomicAdd(G.app_embedding + (size_t)cam * C::APP + i, dcin[C::SH + C::GEO + i]);
          }
        } else if (F.appearance_mode == FNR_APP_MEAN) {
#pragma unroll
          for (int i = 0; i < C::APP; ++i) {
            const float s = warp_sum(dcin[C::SH + C::GEO + i]) / (float)F.num_images;
            if (s != 0.f)
              for (int row = lane; row < F.num_images; row += 32) atomicAdd(G.app_embedding + (size_t)row * C::APP + i, s);
          }
        }
      }
    }
    // ---- base MLP ---------------------------------------------------------------------------
    float denc[C::ENC];
    {
      float dout[C::BASE_OUT];
      dout[0] = kResident ? dout0 : density_grad();
#pragma unroll
      for (int i = 0; i < C::GEO; ++i) dout[1 + i] = d_geo[i];
      if constexpr (kResident) {
        // enc and h1 = relu(base0 enc + b0) again, h1 by the recompute's own row path, so its bits and ReLU mask are the
        // forward's; base1's output is needed only as dout[0]
        load_encoding([&] {
          bool s;
          return field_position(o, d, Rr.starts[pc], Rr.ends[pc], F.position_mode, F.aabb, s);
        });
        Lin::template fwd_relu<kBase0>(P, enc, h1);
        FNR_PHASE(kPhRecompute);
      }
      float dh1[C::BASE_H];
      Lin::template grad_relu<kBase1>(P, G, h1, dout, dh1);
      Lin::template grad<kBase0>(P, G, enc, dh1, denc);
    }
    // ---- hash-table gradient -----------------------------------------------------------------
    if constexpr (kResident) {
      // level_scatter_kernel adds these to the table; streaming stores (one 256 B segment per warp and level) that do
      // not evict the table gradient from L2.  The big family's staged kernel keeps the inline scatter: moving it out
      // made its step slower (DESIGN.md section 4.3).
      if (valid) {
#pragma unroll
        for (int l = 0; l < C::L; ++l) __stcs(B.denc + (size_t)l * N + p, make_float2(denc[2 * l], denc[2 * l + 1]));
      }
    } else if (valid) {
      float2* gt = reinterpret_cast<float2*>(G.hash_table);
#pragma unroll 1
      for (int l = 0; l < C::L; ++l) {
        const float g0 = denc[2 * l], g1 = denc[2 * l + 1];
        if (g0 == 0.f && g1 == 0.f) continue;
        level_scatter(gt, pos, F.scalings[l], l, F.log2T, g0, g1);
      }
    }
    FNR_PHASE(kPhScatter);
  }
  if constexpr (kResident) {
    // every warpgroup, with tiles or without, ends here: one flush of the CTA's weight gradients
    __syncthreads();
#ifdef FNR_BWD_PHASE_TIMERS
    const long long f0 = clock64();
#endif
    Lin::flush_all(G);
#ifdef FNR_BWD_PHASE_TIMERS
    __syncthreads();
    if (threadIdx.x == 0) phase::cycles[0][kPhDwFlush] += (unsigned long long)(clock64() - f0);
#endif
  }
#ifdef FNR_BWD_PHASE_TIMERS
  __syncthreads();  // thread 0's update of the last phase is visible to the threads that flush the counters
  if (threadIdx.x < kBwdPhases) atomicAdd(g_bwd_phase_cycles + threadIdx.x, phase::cycles[0][threadIdx.x] + phase::cycles[1][threadIdx.x]);
#endif
}

#ifdef FNR_BWD_PHASE_TIMERS
// Cycles per backward phase summed over all CTAs since the last call (tools/bench_backward.py --phases); resets them.
extern "C" int fnr_bwd_phase_cycles(unsigned long long* out) {
  static const unsigned long long zero[kBwdPhases] = {};
  cudaError_t e = cudaMemcpyFromSymbol(out, g_bwd_phase_cycles, sizeof(g_bwd_phase_cycles));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_bwd_phase_cycles, zero, sizeof(zero));
  return e == cudaSuccess ? 0 : (int)e;
}
#endif

// ------------------------------------------------------------------------------------------
// K5: level-major hash-table scatter of the small family's tensor-core backward.  A work item is one level of one
// 32-point chunk, taken by one warp; the items are ordered level-major and grid-strided over the warps of persistent CTAs,
// so the whole grid adds level 0 of every point, then level 1, and so on.  A warp's lanes hold consecutive samples of a
// ray, which at the coarse levels often share a cell: warp_level_scatter merges their reds.
// Positions are recomputed with the backward's field_position from the same ray inputs, so the corner rows are the ones
// the simt backward's inline scatter hits.  DESIGN.md section 4.3 has the measured choices (level-major rather than
// all levels of a chunk per work item, one float4 red per x-neighbour pair).
// ------------------------------------------------------------------------------------------
constexpr int kScatterThreads = 256;

__global__ void __launch_bounds__(kScatterThreads) level_scatter_kernel(KField F, KRays Rr, const float2* __restrict__ denc,
                                                                       float2* __restrict__ table_grad) {
  const long long N = (long long)Rr.R * Rr.S;
  const long long chunks = (N + 31) / 32;
  const long long warps = (long long)gridDim.x * (kScatterThreads / 32);
  const int lane = threadIdx.x & 31;
  // w is the same in every lane of a warp: every lane runs every iteration and reaches each shuffle of warp_level_scatter
  // as often as the others.  No lane leaves the loop or skips an iteration on its own; a lane past N or with a zero
  // gradient takes part with active = false.
  for (long long w = ((long long)blockIdx.x * kScatterThreads + threadIdx.x) / 32; w < chunks * F.L; w += warps) {
    const int l = (int)(w / chunks);
    const long long p = (w - l * chunks) * 32 + lane;
    const bool in = p < N;
    const float2 g = in ? __ldcs(denc + (size_t)l * N + p) : make_float2(0.f, 0.f);
    Vec3 pos{0.f, 0.f, 0.f};
    if (in && (g.x != 0.f || g.y != 0.f)) {
      const int r = (int)(p / Rr.S);
      bool sel;
      pos = field_position(Rr.origins + 3 * (size_t)r, Rr.directions + 3 * (size_t)r, Rr.starts[p], Rr.ends[p], F.position_mode,
                           F.aabb, sel);
    }
    warp_level_scatter(table_grad, level_cell(pos, F.scalings[l]), in, l, F.log2T, g.x, g.y, lane);
  }
}

// ------------------------------------------------------------------------------------------
// Export kernel: uniform bins, field in AABB / mean-appearance mode, thresholds + compaction
// (fruit_nerf.py:251-269; export/exporter_utils.py:111-153).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int warp_claim(int* counter, bool pred, int lane, int& rank_out) {
  const unsigned m = __ballot_sync(kFull, pred);
  int basev = 0;
  if (m) {
    const int leader = __ffs(m) - 1;
    if (lane == leader) basev = atomicAdd(counter, __popc(m));
    basev = __shfl_sync(kFull, basev, leader);
  }
  rank_out = __popc(m & ((1u << lane) - 1u));
  return basev;
}

template <class C, bool TC>
__global__ void __launch_bounds__(FieldLayers<C, TC, ForwardPlan>::kThreadsPerCta, FieldLayers<C, TC, ForwardPlan>::kMinCtas)
    simt_export_kernel(KField F, KParams P, KExport E) {
  using Lin = FieldLayers<C, TC, ForwardPlan>;
  constexpr bool kResident = Lin::kResident;
  constexpr int kGroups = Lin::kGroups;
  __shared__ float s_app[C::APP];
  block_mean_embedding(P, F.num_images, C::APP, FNR_APP_MEAN, s_app);
  const int lane = threadIdx.x & 31;
  const long long N = (long long)E.B * E.S;
  // UniformSamplerWithNoise (eval): bins = linspace(0,1,S+1) (made on the host, as the reference does:
  // components/ray_samplers.py:75); t = bins*far + (1-bins)*near
  auto position = [&](long long pc, bool& sel, Vec3& world) {
    const int r = (int)(pc / E.S), s = (int)(pc % E.S);
    const float* bins = E.bins + (size_t)r * E.bins_ray_stride;  // per-ray jittered bins when the stride is S+1
    const float b0 = __ldg(bins + s), b1 = __ldg(bins + s + 1);
    const float t0 = __fadd_rn(__fmul_rn(b0, E.far_plane), __fmul_rn(__fsub_rn(1.0f, b0), E.near_plane));
    const float t1 = __fadd_rn(__fmul_rn(b1, E.far_plane), __fmul_rn(__fsub_rn(1.0f, b1), E.near_plane));
    return field_position(E.origins + 3 * (size_t)r, E.normal, t0, t1, FNR_POS_AABB, F.aabb, sel, &world);
  };
  if constexpr (kResident) {
    const bool mma = mma_warpgroup(F, P, N, nullptr, [&](long long pc) {
      bool sel;
      Vec3 world;
      return position(pc, sel, world);
    });
    if (!mma) return;
  }
  const int g = group_of<kGroups>();
  const unsigned t = thread_of<kGroups>();
  const unsigned span = kResident ? kGroups * kThreads : blockDim.x;  // points of a CTA's round of tiles
  long long k = 0;                                                    // the warpgroup's tile count
  // whole 128-point tiles per warpgroup (see simt_field_forward_kernel): warp-converged row claims, warpgroup-wide MLP layers
  for (long long p0 = (long long)blockIdx.x * span + g * kThreads; p0 < N; p0 += (long long)gridDim.x * span, ++k) {
    const long long p = p0 + t;
    const bool valid = p < N;
    const long long pc = valid ? p : N - 1;
    bool sel;
    Vec3 world;
    const Vec3 pos = position(pc, sel, world);
    float enc[C::ENC];
    if constexpr (kResident)
      resident_encoding(F, P, k, pos, nullptr, enc);
    else
      hash_encode<C::L>(reinterpret_cast<const float2*>(P.hash_table), F.scalings, F.log2T, pos, enc);
    float appv[C::APP];
    load_appearance(P, FNR_APP_MEAN, 0, s_app, appv);
    Acts<C> a;
    field_mlps<C, Lin>(P, enc, E.normal, appv, a);
    const float density = sel ? expf(a.out[0]) : 0.f;
    const float sg = sigmoidf_(a.logit);
    // heaviside(sigmoid(logit) - thr, 0): 1 iff sigmoid - thr > 0
    const int label = (sg - E.label_thr > 0.f) ? 1 : 0;
    if (valid) {
      if (E.sample_density) E.sample_density[p] = density;
      if (E.sample_semantics) E.sample_semantics[p] = a.logit;
      if (E.semantics_colormap) E.semantics_colormap[p] = label;
      if (E.sample_rgb) {
        E.sample_rgb[3 * p] = a.rgb[0];
        E.sample_rgb[3 * p + 1] = a.rgb[1];
        E.sample_rgb[3 * p + 2] = a.rgb[2];
      }
      if (E.point_location) {
        E.point_location[3 * p] = world.x;
        E.point_location[3 * p + 1] = world.y;
        E.point_location[3 * p + 2] = world.z;
      }
    }
    const bool m_den = valid && (density >= E.density_min);
    const bool m_sem = valid && (a.logit >= E.logit_min);
    const bool m_lab = valid && ((float)label >= 0.999f);
    const bool keep[3] = {m_lab && m_den, m_sem && m_den, m_den};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      int rank;
      const int basev = warp_claim(E.counts + k, keep[k], lane, rank);
      if (keep[k] && E.rows[k]) {
        const int row = basev + rank;
        if (row < E.capacity) {
          float* q = E.rows[k] + 7 * (size_t)row;
          q[0] = world.x;
          q[1] = world.y;
          q[2] = world.z;
          q[3] = a.rgb[0];
          q[4] = a.rgb[1];
          q[5] = a.rgb[2];
          q[6] = (k == 2) ? sigmoidf_(density) : sg;
          if (E.keys[k]) E.keys[k][row] = E.point_base + (uint64_t)p;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Hash row export (integer parity hook).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) hash_indices_kernel(KField F, KRays Rr, int32_t* rows, float* positions) {
  const long long N = (long long)Rr.R * Rr.S;
  const uint32_t mask = (1u << F.log2T) - 1u;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(p / Rr.S);
    bool sel;
    const Vec3 pos = field_position(Rr.origins + 3 * (size_t)r, Rr.directions + 3 * (size_t)r, Rr.starts[p], Rr.ends[p],
                                    F.position_mode, F.aabb, sel);
    if (positions) {
      positions[3 * p] = pos.x;
      positions[3 * p + 1] = pos.y;
      positions[3 * p + 2] = pos.z;
    }
    for (int l = 0; l < F.L; ++l) {
      const LevelCell c = level_cell(pos, F.scalings[l]);
      const uint32_t base = (uint32_t)l << F.log2T;
#pragma unroll
      for (int k = 0; k < 8; ++k) rows[((size_t)p * F.L + l) * 8 + k] = (int32_t)corner_row(c, k, mask, base);
    }
  }
}

// ------------------------------------------------------------------------------------------
// Launchers
// ------------------------------------------------------------------------------------------
int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;  // H100 SXM
  }
  return n;
}

int launch_simt_composite(const KRays& Rr, const KComposite& Cm, cudaStream_t st) {
  if (Rr.R == 0) return FNR_OK;
  const int grid = grid_for(Rr.R, kThreads / 32, sm_count() * 16);
  simt_composite_kernel<<<grid, kThreads, 0, st>>>(Rr, Cm);
  return check_launch("simt_composite_kernel");
}

int launch_simt_composite_backward(const KRays& Rr, const KCompositeBwd& B, cudaStream_t st) {
  if (Rr.R == 0) return FNR_OK;
  const int grid = grid_for(Rr.R, kThreads / 32, sm_count() * 16);
  simt_composite_backward_kernel<<<grid, kThreads, 0, st>>>(Rr, B);
  return check_launch("simt_composite_backward_kernel");
}

// One launch of a field kernel over N points on layer type Lin, with `smem` bytes of dynamic shared memory.  Resident
// kernels run one CTA per SM (their shared memory is most of the SM's); the others with dynamic shared memory (the
// backward and every tensor-core instantiation) opt in to it and run as many CTAs as fit on the SMs, and the simt forward
// and export run 16 CTAs per SM.  No more CTAs than the points need (Lin::kGroups warpgroups per CTA, 128 points each).
template <class Lin, class Kernel, class... Args>
static int launch_field(Kernel kernel, int smem, long long N, const char* name, cudaStream_t st, const Args&... args) {
  if (N == 0) return FNR_OK;
  int per_sm = Lin::kResident ? 1 : 16;
  if (smem > 0) {
    // per device: set on every call (cheap), so that a process driving several GPUs opts in on each of them
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute");
    if (!Lin::kResident) {
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, Lin::kThreadsPerCta, smem);
      if (e != cudaSuccess) return check_cuda(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
      if (per_sm < 1) per_sm = 1;
    }
  }
  kernel<<<grid_for(N, Lin::kGroups * kThreads, sm_count() * per_sm), Lin::kThreadsPerCta, smem, st>>>(args...);
  return check_launch(name);
}

// Returns launch(C{}, std::bool_constant<TC>{}) with the family's config C and the implementation TC as types.
template <class Launch>
static auto with_layers(Family fam, bool tc, Launch launch) {
  if (fam == kFamilySmall) return tc ? launch(CfgSmall{}, std::true_type{}) : launch(CfgSmall{}, std::false_type{});
  return tc ? launch(CfgBig{}, std::true_type{}) : launch(CfgBig{}, std::false_type{});
}

int launch_field_forward(Family fam, bool tc, const KField& F, const KParams& P, const KRays& Rr, const KFieldOut& O, cudaStream_t st) {
  return with_layers(fam, tc, [&](auto c, auto t) {
    using C = decltype(c);
    constexpr bool TC = decltype(t)::value;
    using Lin = FieldLayers<C, TC, ForwardPlan>;
    return launch_field<Lin>(simt_field_forward_kernel<C, TC>, Lin::kFwdSmemBytes, (long long)Rr.R * Rr.S,
                             TC ? "simt_field_forward_kernel<wgmma>" : "simt_field_forward_kernel", st, F, P, Rr, O);
  });
}

bool backward_uses_level_scatter(Family fam, bool tc) {
  return with_layers(fam, tc, [](auto c, auto t) { return FieldLayers<decltype(c), decltype(t)::value, BackwardPlan>::kResident; });
}

int launch_field_backward(Family fam, bool tc, const KField& F, const KParams& P, const KParams& G, const KRays& Rr, const KFieldBwd& B,
                          cudaStream_t st) {
  const int rc = with_layers(fam, tc, [&](auto c, auto t) {
    using C = decltype(c);
    constexpr bool TC = decltype(t)::value;
    using Lin = FieldLayers<C, TC, BackwardPlan>;
    return launch_field<Lin>(simt_field_backward_kernel<C, TC>, Lin::kBwdSmemBytes, (long long)Rr.R * Rr.S,
                             TC ? "simt_field_backward_kernel<wgmma>" : "simt_field_backward_kernel", st, F, P, G, Rr, B);
  });
  if (rc || !backward_uses_level_scatter(fam, tc)) return rc;
  return launch_level_scatter(F, Rr, B.denc, reinterpret_cast<float2*>(G.hash_table), st);
}

int launch_level_scatter(const KField& F, const KRays& Rr, const float2* denc, float2* table_grad, cudaStream_t st) {
  const long long N = (long long)Rr.R * Rr.S;
  if (N == 0) return FNR_OK;
  // persistent CTAs, as many as are resident at once
  static int per_sm = 0;
  if (!per_sm) {
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, level_scatter_kernel, kScatterThreads, 0);
    if (e != cudaSuccess) return check_cuda(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    if (per_sm < 1) per_sm = 1;
  }
  level_scatter_kernel<<<grid_for((N + 31) / 32 * F.L, kScatterThreads / 32, sm_count() * per_sm), kScatterThreads, 0, st>>>(
      F, Rr, denc, table_grad);
  return check_launch("level_scatter_kernel");
}

int launch_export(Family fam, bool tc, const KField& F, const KParams& P, const KExport& E, cudaStream_t st) {
  return with_layers(fam, tc, [&](auto c, auto t) {
    using C = decltype(c);
    constexpr bool TC = decltype(t)::value;
    using Lin = FieldLayers<C, TC, ForwardPlan>;
    return launch_field<Lin>(simt_export_kernel<C, TC>, Lin::kFwdSmemBytes, (long long)E.B * E.S,
                             TC ? "simt_export_kernel<wgmma>" : "simt_export_kernel", st, F, P, E);
  });
}

int launch_hash_indices(const KField& F, const KRays& Rr, int32_t* rows, float* positions, cudaStream_t st) {
  const long long N = (long long)Rr.R * Rr.S;
  if (N == 0) return FNR_OK;
  const int grid = grid_for(N, kThreads, sm_count() * 16);
  hash_indices_kernel<<<grid, kThreads, 0, st>>>(F, Rr, rows, positions);
  return check_launch("hash_indices_kernel");
}

}  // namespace fnr
