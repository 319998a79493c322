// Kernels of the FruitNeRF hot path: one thread per sample point, per-ray compositing by one warp per ray.
//
// The field kernels (forward, export, backward) are instantiated twice through Layers<C, TC>.  TC = false is the "simt"
// implementation, the exact-fp32 device path: MLP weights read straight from the torch parameter tensors through the
// read-only path (warp-uniform addresses, float4 where the row alignment allows); it is the on-device fp32 reference
// the tensor-core path is checked against at full size.  TC = true runs the MLP layers block-wide on the Hopper tensor
// cores (fnr_wgmma.cuh).
//
// Reference semantics: fruit_nerf/fruit_field.py:168-301, fruit_nerf/fruit_nerf.py:251-269,316-357.
#include <type_traits>
#include "fnr_common.cuh"
#include "fnr_kernels.h"
#include "fnr_wgmma.cuh"

namespace fnr {

constexpr int kThreads = 128;

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

// How the field kernels evaluate a Linear layer W [N][K]: forward y = act(W x + b), input gradient dx = W^T dy and
// weight gradient dW = dY^T X over the CTA's tile.  TC = false: per thread in fp32 on the CUDA cores (the exact device
// reference).  TC = true: block-wide on the tensor cores (fnr_wgmma.cuh; every thread of the 128-thread CTA must take part).
template <class C, bool TC>
struct Layers {
  // the 1- and 3-wide output heads (64 MACs per point) stay in exact fp32 on the CUDA cores on both paths
  static constexpr bool tensor(int n) { return TC && n >= 8; }
  // dynamic shared memory: the sX / sY tiles of tile_weight_grad, and the wgmma operand plans (the backward's heads
  // still use tile_weight_grad, so its tensor-core plan holds that tile too)
  static constexpr int kTileBytes = 2 * kThreads * (((C::MAXW + 3) & ~3) + 4) * 4;
  static constexpr int kFwdSmemBytes = TC ? wg::Smem<C::MAXW, C::MAXW>::kBytes : 0;
  static constexpr int kBwdSmemBytes =
      TC ? cmax(cmax(wg::Smem<C::MAXW, C::MAXW>::kBytes, wg::DwSmem<C::MAXW, C::MAXW>::kBytes), kTileBytes) : kTileBytes;

  static __device__ __forceinline__ uint8_t* dyn_smem() {
    extern __shared__ __align__(128) uint8_t wg_smem[];
    return wg_smem;
  }
  template <int K, int N, bool RELU>
  static __device__ __forceinline__ void fwd(const float* __restrict__ W, const float* __restrict__ b, const float (&x)[K], float (&y)[N]) {
    if constexpr (tensor(N))
      wg::linear<C::MAXW, C::MAXW, K, N, RELU>(dyn_smem(), W, b, x, y);
    else
      linear_fwd<K, N, RELU>(W, b, x, y);
  }
  template <int K, int N>
  static __device__ __forceinline__ void dx(const float* __restrict__ W, const float (&dy)[N], float (&dxv)[K]) {
    if constexpr (tensor(N))
      wg::linear_dx<C::MAXW, C::MAXW, K, N>(dyn_smem(), W, dy, dxv);
    else
      linear_bwd_input<K, N>(W, dy, dxv);
    FNR_PHASE(kPhDx);
  }
  template <int K, int N>
  static __device__ __forceinline__ void dw(float* sX, float* sY, const float (&x)[K], const float (&dy)[N], float* gW, float* gb) {
    if constexpr (tensor(N))
      wg::weight_grad<K, N>(dyn_smem(), x, dy, gW, gb);
    else
      tile_weight_grad<K, N>(sX, sY, x, dy, gW, gb);
    FNR_PHASE(kPhDw);
  }
};

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
// base MLP: enc -> [h0, geo...]; geo = out[1:]
template <class C, bool TC>
__device__ __forceinline__ void base_fwd(const KParams& P, const float (&enc)[C::ENC], float (&h1)[C::BASE_H],
                                         float (&out)[C::BASE_OUT], float (&geo)[C::GEO]) {
  using Lin = Layers<C, TC>;
  Lin::template fwd<C::ENC, C::BASE_H, true>(P.base_w[0], P.base_b[0], enc, h1);
  Lin::template fwd<C::BASE_H, C::BASE_OUT, false>(P.base_w[1], P.base_b[1], h1, out);
#pragma unroll
  for (int i = 0; i < C::GEO; ++i) geo[i] = out[1 + i];
}

// semantic branch up to the logit head: mlp_semantics(detach(geo)) (fruit_field.py:263-268)
template <class C, bool TC>
__device__ __forceinline__ void semantic_fwd(const KParams& P, const float (&geo)[C::GEO], float (&z1)[C::SEM_H],
                                             float (&z2)[C::SEM_LAYERS == 3 ? C::SEM_H : 1], float (&zo)[C::SEM_OUT]) {
  using Lin = Layers<C, TC>;
  Lin::template fwd<C::GEO, C::SEM_H, true>(P.sem_w[0], P.sem_b[0], geo, z1);
  if constexpr (C::SEM_LAYERS == 3) {
    Lin::template fwd<C::SEM_H, C::SEM_H, true>(P.sem_w[1], P.sem_b[1], z1, z2);
    Lin::template fwd<C::SEM_H, C::SEM_OUT, false>(P.sem_w[2], P.sem_b[2], z2, zo);
  } else {
    Lin::template fwd<C::SEM_H, C::SEM_OUT, false>(P.sem_w[1], P.sem_b[1], z1, zo);
  }
}

// colour branch up to the sigmoid: cat[SH(dir), geo, appearance] -> MLP (fruit_field.py:270-278)
template <class C, bool TC>
__device__ __forceinline__ void colour_fwd(const KParams& P, const float* __restrict__ dir, const float (&geo)[C::GEO],
                                           const float (&app)[C::APP], float (&cin)[C::COL_IN], float (&c1)[C::COL_H],
                                           float (&c2)[C::COL_H], float (&o3)[3]) {
  using Lin = Layers<C, TC>;
  sh_degree4(dir[0], dir[1], dir[2], cin);
#pragma unroll
  for (int i = 0; i < C::GEO; ++i) cin[C::SH + i] = geo[i];
#pragma unroll
  for (int i = 0; i < C::APP; ++i) cin[C::SH + C::GEO + i] = app[i];
  Lin::template fwd<C::COL_IN, C::COL_H, true>(P.col_w[0], P.col_b[0], cin, c1);
  Lin::template fwd<C::COL_H, C::COL_H, true>(P.col_w[1], P.col_b[1], c1, c2);
  Lin::template fwd<C::COL_H, 3, false>(P.col_w[2], P.col_b[2], c2, o3);
}

template <class C, bool TC>
__device__ __forceinline__ void field_mlps(const KParams& P, const float (&enc)[C::ENC], const float* __restrict__ dir,
                                           const float (&app)[C::APP], Acts<C>& a) {
  float geo[C::GEO];
  base_fwd<C, TC>(P, enc, a.h1, a.out, geo);
  semantic_fwd<C, TC>(P, geo, a.z1, a.z2, a.zo);
  float lg[1];
  Layers<C, TC>::template fwd<C::SEM_OUT, 1, false>(P.head_w, P.head_b, a.zo, lg);
  a.logit = lg[0];
  float o3[3];
  colour_fwd<C, TC>(P, dir, geo, app, a.cin, a.c1, a.c2, o3);
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
// The loop runs whole 128-point tiles per CTA (threads past N compute a clamped point and store nothing), so that the
// block-wide tensor-core layers see every thread.
template <class C, bool TC>
__global__ void __launch_bounds__(kThreads) simt_field_forward_kernel(KField F, KParams P, KRays Rr, KFieldOut O) {
  __shared__ float s_app[C::APP];
  block_mean_embedding(P, F.num_images, C::APP, F.appearance_mode, s_app);
  const long long N = (long long)Rr.R * Rr.S;
  for (long long p0 = (long long)blockIdx.x * blockDim.x; p0 < N; p0 += (long long)gridDim.x * blockDim.x) {
    const bool valid = p0 + threadIdx.x < N;
    const long long p = valid ? p0 + threadIdx.x : N - 1;
    const int r = (int)(p / Rr.S);
    const float* o = Rr.origins + 3 * (size_t)r;
    const float* d = Rr.directions + 3 * (size_t)r;
    bool sel;
    const Vec3 pos = field_position(o, d, Rr.starts[p], Rr.ends[p], F.position_mode, F.aabb, sel);
    float enc[C::ENC];
    hash_encode<C::L>(reinterpret_cast<const float2*>(P.hash_table), F.scalings, F.log2T, pos, enc);
    if (O.stash_encoding && valid) {
      float4* st = reinterpret_cast<float4*>(O.stash_encoding + (size_t)p * C::ENC);
#pragma unroll
      for (int i = 0; i < C::ENC / 4; ++i) st[i] = make_float4(enc[4 * i], enc[4 * i + 1], enc[4 * i + 2], enc[4 * i + 3]);
    }
    // not load_appearance: selecting the source row once compiles to ~130 fewer instructions in this kernel
    const float* app = (F.appearance_mode == FNR_APP_PER_CAMERA)
                           ? P.app_embedding + (size_t)Rr.camera_indices[r] * C::APP
                           : s_app;
    float appv[C::APP];
#pragma unroll
    for (int i = 0; i < C::APP; ++i) appv[i] = (F.appearance_mode == FNR_APP_PER_CAMERA) ? __ldg(app + i) : app[i];
    Acts<C> a;
    field_mlps<C, TC>(P, enc, d, appv, a);
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
// K4: per-point field backward.  Weight gradients: the CTA's 128 points form one tile; for every
// layer the tile's inputs X[128,K] and output grads dY[128,N] go to shared memory and each thread
// reduces a 4x4 block of dW = dY^T X over the tile, then adds it to the global gradient.
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
__global__ void __launch_bounds__(kThreads) simt_field_backward_kernel(KField F, KParams P, KParams G, KRays Rr,
                                                                      KFieldBwd B) {
  using Lin = Layers<C, TC>;
  extern __shared__ __align__(16) float smem[];
  constexpr int TP = ((C::MAXW + 3) & ~3) + 4;
  float* sX = smem;
  float* sY = smem + kThreads * TP;
  __shared__ float s_app[C::APP];
  block_mean_embedding(P, F.num_images, C::APP, F.appearance_mode, s_app);
#ifdef FNR_BWD_PHASE_TIMERS
  if (threadIdx.x < kBwdPhases) phase::cycles[threadIdx.x] = 0;
  if (threadIdx.x == 0) phase::last = clock64();
#endif
  const long long N = (long long)Rr.R * Rr.S;
  const long long tiles = (N + kThreads - 1) / kThreads;
  const int lane = threadIdx.x & 31;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long p = tile * kThreads + threadIdx.x;
    const bool valid = p < N;
    const long long pc = valid ? p : N - 1;
    const int r = (int)(pc / Rr.S);
    const float* o = Rr.origins + 3 * (size_t)r;
    const float* d = Rr.directions + 3 * (size_t)r;
    bool sel;
    const Vec3 pos = field_position(o, d, Rr.starts[pc], Rr.ends[pc], F.position_mode, F.aabb, sel);
    float enc[C::ENC];
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
      hash_encode<C::L>(reinterpret_cast<const float2*>(P.hash_table), F.scalings, F.log2T, pos, enc);
    }
    const int cam = (F.appearance_mode == FNR_APP_PER_CAMERA) ? Rr.camera_indices[r] : 0;
    float appv[C::APP];
    load_appearance(P, F.appearance_mode, cam, s_app, appv);
    // upstream per-point grads (zero for padding threads)
    const float* pg = B.point_grads + 5 * (size_t)pc;
    const float vm = valid ? 1.f : 0.f;
    const float d_sigma = pg[0] * vm;
    const float d_rgb[3] = {pg[1] * vm, pg[2] * vm, pg[3] * vm};
    const float d_logit = pg[4] * vm;
    FNR_PHASE(kPhLoad);

    // The forward is recomputed branch by branch with field_mlps' branch functions, and each branch is back-propagated
    // right after its forward: only the base MLP's activations live across the whole tile.
    float h1[C::BASE_H], out[C::BASE_OUT], geo[C::GEO];
    base_fwd<C, TC>(P, enc, h1, out, geo);
    FNR_PHASE(kPhRecompute);

    float d_geo[C::GEO];
#pragma unroll
    for (int i = 0; i < C::GEO; ++i) d_geo[i] = 0.f;

    // ---- semantic branch (its logit head is not needed: d_logit is the upstream gradient) ------------------------
    {
      float z1[C::SEM_H], zo[C::SEM_OUT];
      float z2[C::SEM_LAYERS == 3 ? C::SEM_H : 1];
      semantic_fwd<C, TC>(P, geo, z1, z2, zo);
      FNR_PHASE(kPhRecompute);
      float dlg[1] = {d_logit};
      float dzo[C::SEM_OUT];
      Lin::template dx<C::SEM_OUT, 1>(P.head_w, dlg, dzo);
      Lin::template dw<C::SEM_OUT, 1>(sX, sY, zo, dlg, G.head_w, G.head_b);
      float dz1[C::SEM_H];
      if constexpr (C::SEM_LAYERS == 3) {
        float dz2[C::SEM_H];
        Lin::template dx<C::SEM_H, C::SEM_OUT>(P.sem_w[2], dzo, dz2);
        Lin::template dw<C::SEM_H, C::SEM_OUT>(sX, sY, z2, dzo, G.sem_w[2], G.sem_b[2]);
#pragma unroll
        for (int i = 0; i < C::SEM_H; ++i) dz2[i] = z2[i] > 0.f ? dz2[i] : 0.f;
        Lin::template dx<C::SEM_H, C::SEM_H>(P.sem_w[1], dz2, dz1);
        Lin::template dw<C::SEM_H, C::SEM_H>(sX, sY, z1, dz2, G.sem_w[1], G.sem_b[1]);
      } else {
        Lin::template dx<C::SEM_H, C::SEM_OUT>(P.sem_w[1], dzo, dz1);
        Lin::template dw<C::SEM_H, C::SEM_OUT>(sX, sY, z1, dzo, G.sem_w[1], G.sem_b[1]);
      }
#pragma unroll
      for (int i = 0; i < C::SEM_H; ++i) dz1[i] = z1[i] > 0.f ? dz1[i] : 0.f;
      Lin::template dw<C::GEO, C::SEM_H>(sX, sY, geo, dz1, G.sem_w[0], G.sem_b[0]);
      if (F.pass_semantic_gradients) {
        float dg[C::GEO];
        Lin::template dx<C::GEO, C::SEM_H>(P.sem_w[0], dz1, dg);
#pragma unroll
        for (int i = 0; i < C::GEO; ++i) d_geo[i] += dg[i];
      }
    }
    // ---- colour branch ---------------------------------------------------------------------
    {
      float cin[C::COL_IN], c1[C::COL_H], c2[C::COL_H], o3[3];
      colour_fwd<C, TC>(P, d, geo, appv, cin, c1, c2, o3);
      FNR_PHASE(kPhRecompute);
      float do3[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const float rgb = sigmoidf_(o3[i]);
        do3[i] = d_rgb[i] * rgb * (1.0f - rgb);
      }
      float dc2[C::COL_H], dc1[C::COL_H], dcin[C::COL_IN];
      Lin::template dx<C::COL_H, 3>(P.col_w[2], do3, dc2);
      Lin::template dw<C::COL_H, 3>(sX, sY, c2, do3, G.col_w[2], G.col_b[2]);
#pragma unroll
      for (int i = 0; i < C::COL_H; ++i) dc2[i] = c2[i] > 0.f ? dc2[i] : 0.f;
      Lin::template dx<C::COL_H, C::COL_H>(P.col_w[1], dc2, dc1);
      Lin::template dw<C::COL_H, C::COL_H>(sX, sY, c1, dc2, G.col_w[1], G.col_b[1]);
#pragma unroll
      for (int i = 0; i < C::COL_H; ++i) dc1[i] = c1[i] > 0.f ? dc1[i] : 0.f;
      Lin::template dx<C::COL_IN, C::COL_H>(P.col_w[0], dc1, dcin);
      Lin::template dw<C::COL_IN, C::COL_H>(sX, sY, cin, dc1, G.col_w[0], G.col_b[0]);
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
    // ---- base MLP ---------------------------------------------------------------------------
    float denc[C::ENC];
    {
      float dout[C::BASE_OUT];
      // trunc_exp backward: g * exp(clamp(x, -15, 15)); density = exp(h0) * selector
      dout[0] = sel ? d_sigma * expf(fminf(fmaxf(out[0], -15.f), 15.f)) : 0.f;
#pragma unroll
      for (int i = 0; i < C::GEO; ++i) dout[1 + i] = d_geo[i];
      float dh1[C::BASE_H];
      Lin::template dx<C::BASE_H, C::BASE_OUT>(P.base_w[1], dout, dh1);
      Lin::template dw<C::BASE_H, C::BASE_OUT>(sX, sY, h1, dout, G.base_w[1], G.base_b[1]);
#pragma unroll
      for (int i = 0; i < C::BASE_H; ++i) dh1[i] = h1[i] > 0.f ? dh1[i] : 0.f;
      Lin::template dx<C::ENC, C::BASE_H>(P.base_w[0], dh1, denc);
      Lin::template dw<C::ENC, C::BASE_H>(sX, sY, enc, dh1, G.base_w[0], G.base_b[0]);
    }
    // ---- hash-table scatter -----------------------------------------------------------------
    if (valid) {
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
#ifdef FNR_BWD_PHASE_TIMERS
  __syncthreads();  // thread 0's update of the last phase is visible to the threads that flush the counters
  if (threadIdx.x < kBwdPhases) atomicAdd(g_bwd_phase_cycles + threadIdx.x, phase::cycles[threadIdx.x]);
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
__global__ void __launch_bounds__(kThreads) simt_export_kernel(KField F, KParams P, KExport E) {
  __shared__ float s_app[C::APP];
  block_mean_embedding(P, F.num_images, C::APP, FNR_APP_MEAN, s_app);
  const int lane = threadIdx.x & 31;
  const long long N = (long long)E.B * E.S;
  // whole 128-point tiles per CTA (see simt_field_forward_kernel): warp-converged row claims, block-wide MLP layers
  for (long long p0 = (long long)blockIdx.x * blockDim.x; p0 < N; p0 += (long long)gridDim.x * blockDim.x) {
    const long long p = p0 + threadIdx.x;
    const bool valid = p < N;
    const long long pc = valid ? p : N - 1;
    const int r = (int)(pc / E.S), s = (int)(pc % E.S);
    // UniformSamplerWithNoise (eval): bins = linspace(0,1,S+1) (made on the host, as the
    // reference does: components/ray_samplers.py:75); t = bins*far + (1-bins)*near
    const float* bins = E.bins + (size_t)r * E.bins_ray_stride;  // per-ray jittered bins when the stride is S+1
    const float b0 = __ldg(bins + s), b1 = __ldg(bins + s + 1);
    const float t0 = __fadd_rn(__fmul_rn(b0, E.far_plane), __fmul_rn(__fsub_rn(1.0f, b0), E.near_plane));
    const float t1 = __fadd_rn(__fmul_rn(b1, E.far_plane), __fmul_rn(__fsub_rn(1.0f, b1), E.near_plane));
    const float* o = E.origins + 3 * (size_t)r;
    bool sel;
    Vec3 world;
    const Vec3 pos = field_position(o, E.normal, t0, t1, FNR_POS_AABB, F.aabb, sel, &world);
    float enc[C::ENC];
    hash_encode<C::L>(reinterpret_cast<const float2*>(P.hash_table), F.scalings, F.log2T, pos, enc);
    float appv[C::APP];
    load_appearance(P, FNR_APP_MEAN, 0, s_app, appv);
    Acts<C> a;
    field_mlps<C, TC>(P, enc, E.normal, appv, a);
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

// One launch of a field kernel over N points.  Kernels with dynamic shared memory (the backward and every tensor-core
// instantiation) opt in to it and run as many CTAs as fit on the SMs; the simt forward and export run 16 CTAs per SM.
template <class Kernel, class... Args>
static int launch_field_kernel(Kernel kernel, int smem, long long N, const char* name, cudaStream_t st, const Args&... args) {
  if (N == 0) return FNR_OK;
  int per_sm = 16;
  if (smem > 0) {
    // per device: set on every call (cheap), so that a process driving several GPUs opts in on each of them
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute");
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem);
    if (e != cudaSuccess) return check_cuda(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    if (per_sm < 1) per_sm = 1;
  }
  kernel<<<grid_for(N, kThreads, sm_count() * per_sm), kThreads, smem, st>>>(args...);
  return check_launch(name);
}

// Calls launch(C{}, std::bool_constant<TC>{}) with the family's config C and the implementation TC as types.
template <class Launch>
static int with_layers(Family fam, bool tc, Launch launch) {
  if (fam == kFamilySmall) return tc ? launch(CfgSmall{}, std::true_type{}) : launch(CfgSmall{}, std::false_type{});
  return tc ? launch(CfgBig{}, std::true_type{}) : launch(CfgBig{}, std::false_type{});
}

int launch_field_forward(Family fam, bool tc, const KField& F, const KParams& P, const KRays& Rr, const KFieldOut& O, cudaStream_t st) {
  return with_layers(fam, tc, [&](auto c, auto t) {
    using C = decltype(c);
    constexpr bool TC = decltype(t)::value;
    return launch_field_kernel(simt_field_forward_kernel<C, TC>, Layers<C, TC>::kFwdSmemBytes, (long long)Rr.R * Rr.S,
                               TC ? "simt_field_forward_kernel<wgmma>" : "simt_field_forward_kernel", st, F, P, Rr, O);
  });
}

int launch_field_backward(Family fam, bool tc, const KField& F, const KParams& P, const KParams& G, const KRays& Rr, const KFieldBwd& B,
                          cudaStream_t st) {
  return with_layers(fam, tc, [&](auto c, auto t) {
    using C = decltype(c);
    constexpr bool TC = decltype(t)::value;
    return launch_field_kernel(simt_field_backward_kernel<C, TC>, Layers<C, TC>::kBwdSmemBytes, (long long)Rr.R * Rr.S,
                               TC ? "simt_field_backward_kernel<wgmma>" : "simt_field_backward_kernel", st, F, P, G, Rr, B);
  });
}

int launch_export(Family fam, bool tc, const KField& F, const KParams& P, const KExport& E, cudaStream_t st) {
  return with_layers(fam, tc, [&](auto c, auto t) {
    using C = decltype(c);
    constexpr bool TC = decltype(t)::value;
    return launch_field_kernel(simt_export_kernel<C, TC>, Layers<C, TC>::kFwdSmemBytes, (long long)E.B * E.S,
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
