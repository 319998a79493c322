// Proposal-sampling stage of the nerfacto-style sampler FruitNeRF trains with
// (fruit_nerf/fruit_nerf.py:104-158, 318; SURVEY.md section 8a row A13):
//   proposal_weights   nerfstudio HashMLPDensityField.get_density (small hash grid -> Linear/ReLU/Linear ->
//                      trunc_exp * selector) fused with RaySamples.get_weights, one warp per ray
//   pdf_sample         nerfstudio PDFSampler (histogram padding, cdf, searchsorted right, lerp) + the
//                      piecewise-linear-in-disparity spacing -> euclidean map, one warp per ray
//   interlevel_loss    nerfstudio losses.interlevel_loss (lossfun_outer) forward + gradient w.r.t. the
//                      proposal weights, one warp per ray
// fp32 CUDA-core kernels: the proposal MLP is 10 -> 16 -> 1 (176 MAC / sample); the work is gathers + scans.
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kHidden = 16;
constexpr int kMaxLevels = 8;
constexpr int kWarpsPerBlock = 4;

struct PropNet {  // shared-memory copy of the tiny MLP
  float w0[kHidden][2 * kMaxLevels];
  float b0[kHidden];
  float w1[kHidden];
  float b1;
};

__device__ __forceinline__ void load_net(PropNet& n, const KDensity& D) {
  const int in = 2 * D.L;
  for (int i = threadIdx.x; i < kHidden * in; i += blockDim.x) n.w0[i / in][i % in] = __ldg(D.w0 + i);
  for (int i = threadIdx.x; i < kHidden; i += blockDim.x) {
    n.b0[i] = __ldg(D.b0 + i);
    n.w1[i] = __ldg(D.w1 + i);
  }
  if (threadIdx.x == 0) n.b1 = __ldg(D.b1);
  __syncthreads();
}

// position of a sample in [0,1]^3 (same op order as the main field) and its selector
__device__ __forceinline__ Vec3 prop_position(const KDensity& D, const float* o, const float* d, float start, float end, bool& sel) {
  return field_position(o, d, start, end, D.position_mode, D.aabb, sel);
}

// encode + MLP.  enc / hid are kept for the backward.
__device__ __forceinline__ float prop_mlp(const KDensity& D, const PropNet& n, const Vec3& p, float (&enc)[2 * kMaxLevels], float (&hid)[kHidden]) {
  const float2* table = reinterpret_cast<const float2*>(D.hash_table);
#pragma unroll
  for (int l = 0; l < kMaxLevels; ++l) {
    if (l < D.L) {
      const float2 r = level_gather(table, p, D.scalings[l], l, D.log2T);
      enc[2 * l] = r.x;
      enc[2 * l + 1] = r.y;
    } else {
      enc[2 * l] = 0.f;
      enc[2 * l + 1] = 0.f;
    }
  }
  float out = n.b1;
#pragma unroll
  for (int j = 0; j < kHidden; ++j) {
    float a = n.b0[j];
#pragma unroll
    for (int k = 0; k < 2 * kMaxLevels; ++k)
      if (k < 2 * D.L) a = fmaf(n.w0[j][k], enc[k], a);
    hid[j] = fmaxf(a, 0.f);
    out = fmaf(n.w1[j], hid[j], out);
  }
  return out;
}

// ---- forward: density + weights ------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * kWarpsPerBlock) proposal_weights_forward_kernel(KDensity D, KRays Rr, float* __restrict__ density,
                                                                                   float* __restrict__ weights) {
  __shared__ PropNet net;
  load_net(net, D);
  const int lane = threadIdx.x & 31;
  const int S = Rr.S;
  for (int r = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); r < Rr.R; r += gridDim.x * kWarpsPerBlock) {
    const float* o = Rr.origins + 3 * (size_t)r;
    const float* d = Rr.directions + 3 * (size_t)r;
    const size_t base = (size_t)r * S;
    float run_x = 0.f;
    for (int c0 = 0; c0 < S; c0 += 32) {
      const int i = c0 + lane;
      const bool in = i < S;
      float x = 0.f, sigma = 0.f;
      if (in) {
        const float st = Rr.starts[base + i], en = Rr.ends[base + i];
        bool sel;
        const Vec3 p = prop_position(D, o, d, st, en, sel);
        float enc[2 * kMaxLevels], hid[kHidden];
        const float h = prop_mlp(D, net, p, enc, hid);
        sigma = sel ? expf(h) : 0.f;
        if (density) density[base + i] = sigma;
        x = (en - st) * sigma;
      }
      const float w = chunk_weight(x, in, lane, run_x);
      if (in) weights[base + i] = w;
    }
  }
}

// ---- backward: d_weights -> d_density -> MLP / hash-table gradients -------------------------------------
struct PropGradAcc {  // per-CTA accumulators of the tiny MLP's gradients
  float w0[kHidden][2 * kMaxLevels];
  float b0[kHidden];
  float w1[kHidden];
  float b1;
};

__global__ void __launch_bounds__(32 * kWarpsPerBlock) proposal_weights_backward_kernel(KDensity D, KDensity G, KRays Rr,
                                                                                    const float* __restrict__ density,
                                                                                    const float* __restrict__ weights,
                                                                                    const float* __restrict__ d_weights) {
  __shared__ PropNet net;
  __shared__ PropGradAcc acc;
  for (int i = threadIdx.x; i < (int)(sizeof(PropGradAcc) / 4); i += blockDim.x) reinterpret_cast<float*>(&acc)[i] = 0.f;
  load_net(net, D);
  const int lane = threadIdx.x & 31;
  const int S = Rr.S;
  float2* gtab = reinterpret_cast<float2*>(G.hash_table);
  for (int r = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); r < Rr.R; r += gridDim.x * kWarpsPerBlock) {
    const float* o = Rr.origins + 3 * (size_t)r;
    const float* d = Rr.directions + 3 * (size_t)r;
    const size_t base = (size_t)r * S;
    const float later_chunks = later_chunks_sum(S, lane, [&](int i) { return d_weights[base + i] * weights[base + i]; });
    float run_x = 0.f;
    for (int c0 = 0, ci = 0; c0 < S; c0 += 32, ++ci) {
      const int i = c0 + lane;
      const bool in = i < S;
      float x = 0.f, Gi = 0.f, w = 0.f, delta = 0.f, st = 0.f, en = 0.f;
      if (in) {
        st = Rr.starts[base + i];
        en = Rr.ends[base + i];
        delta = en - st;
        x = delta * density[base + i];
        w = weights[base + i];
        Gi = d_weights[base + i];
      }
      const float xin = warp_incl_scan(x, lane);
      const float suffix = chunk_suffix(Gi * w, later_chunks, ci, lane);
      float dh = 0.f;
      float enc[2 * kMaxLevels], hid[kHidden];
      Vec3 p = {0.f, 0.f, 0.f};
      bool sel = false;
#pragma unroll
      for (int k = 0; k < 2 * kMaxLevels; ++k) enc[k] = 0.f;
#pragma unroll
      for (int j = 0; j < kHidden; ++j) hid[j] = 0.f;
      if (in) {
        const float dsig = weights_dsigma(delta, Gi, run_x, xin, suffix);
        p = prop_position(D, o, d, st, en, sel);
        const float h = prop_mlp(D, net, p, enc, hid);
        dh = sel ? dsig * expf(fminf(fmaxf(h, -15.f), 15.f)) : 0.f;  // trunc_exp backward
      }
      run_x += __shfl_sync(kFull, xin, 31);
      // MLP backward (per lane), gradients reduced over the warp into the CTA accumulators
      float dhid[kHidden];
#pragma unroll
      for (int j = 0; j < kHidden; ++j) dhid[j] = hid[j] > 0.f ? dh * net.w1[j] : 0.f;
      {
        const float s = warp_sum(dh);
        if (lane == 0 && s != 0.f) atomicAdd(&acc.b1, s);
      }
#pragma unroll
      for (int j = 0; j < kHidden; ++j) {
        const float s1 = warp_sum(dh * hid[j]);
        const float s0 = warp_sum(dhid[j]);
        if (lane == 0) {
          if (s1 != 0.f) atomicAdd(&acc.w1[j], s1);
          if (s0 != 0.f) atomicAdd(&acc.b0[j], s0);
        }
      }
      // dW0[j][k] = sum_lanes dhid[j] * enc[k]: lane k (< 2L) collects column k
      const int in_dim = 2 * D.L;
#pragma unroll
      for (int j = 0; j < kHidden; ++j) {
        float mine = 0.f;
#pragma unroll
        for (int k = 0; k < 2 * kMaxLevels; ++k) {
          const float s = warp_sum(dhid[j] * enc[k]);
          if (lane == k) mine = s;
        }
        if (lane < in_dim && mine != 0.f) atomicAdd(&acc.w0[j][lane], mine);
      }
      // encoding gradient -> hash-table scatter
      if (in && dh != 0.f) {
#pragma unroll
        for (int l = 0; l < kMaxLevels; ++l) {
          if (l < D.L) {
            float g0 = 0.f, g1 = 0.f;
#pragma unroll
            for (int j = 0; j < kHidden; ++j) {
              g0 = fmaf(net.w0[j][2 * l], dhid[j], g0);
              g1 = fmaf(net.w0[j][2 * l + 1], dhid[j], g1);
            }
            level_scatter(gtab, p, D.scalings[l], l, D.log2T, g0, g1);
          }
        }
      }
    }
  }
  __syncthreads();
  const int in_dim = 2 * D.L;
  for (int i = threadIdx.x; i < kHidden * in_dim; i += blockDim.x) {
    const float v = acc.w0[i / in_dim][i % in_dim];
    if (v != 0.f) atomicAdd(G.w0 + i, v);
  }
  for (int i = threadIdx.x; i < kHidden; i += blockDim.x) {
    if (acc.b0[i] != 0.f) atomicAdd(G.b0 + i, acc.b0[i]);
    if (acc.w1[i] != 0.f) atomicAdd(G.w1 + i, acc.w1[i]);
  }
  if (threadIdx.x == 0 && acc.b1 != 0.f) atomicAdd(G.b1, acc.b1);
}

// ---- PDF sampler -------------------------------------------------------------------------------------
__device__ __forceinline__ float lindisp_fn(float x) { return x < 1.f ? x / 2.f : 1.f - 1.f / (2.f * x); }
__device__ __forceinline__ float lindisp_inv(float x) { return x < 0.5f ? 2.f * x : 1.f / (2.f - 2.f * x); }

constexpr int kMaxPdfBins = 1024;

__global__ void __launch_bounds__(32 * kWarpsPerBlock) pdf_sample_kernel(KPdf A) {
  __shared__ float s_cdf[kWarpsPerBlock][kMaxPdfBins + 1];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int S = A.S, NB = A.num_samples + 1;
  float* cdf = s_cdf[wib];
  for (int r = blockIdx.x * kWarpsPerBlock + wib; r < A.R; r += gridDim.x * kWarpsPerBlock) {
    const float* w = A.weights + (size_t)r * S;
    const float* eb = A.existing_bins + (size_t)r * (S + 1);
    const float anneal = A.anneal_dev ? __ldg(A.anneal_dev) : A.anneal;
    // weights^anneal + histogram padding, then the zero-weight guard of the reference
    float part = 0.f;
    for (int i = lane; i < S; i += 32) {
      float v = w[i];
      if (anneal != 1.0f) v = powf(v, anneal);
      part += v + A.hist_padding;
    }
    float wsum = warp_sum(part);
    const float padding = fmaxf(A.eps - wsum, 0.f);
    wsum += padding;
    const float pad_each = padding / (float)S;
    if (lane == 0) cdf[0] = 0.f;
    warp_cumsum(
        S, lane,
        [=](int i) {
          float v = w[i];
          if (anneal != 1.0f) v = powf(v, anneal);
          return (v + A.hist_padding + pad_each) / wsum;
        },
        [=](int i, float c) { cdf[i + 1] = fminf(1.0f, c); });
    __syncwarp();
    const float near_s = lindisp_fn(A.nears[r]), far_s = lindisp_fn(A.fars[r]);
    float* out_bins = A.new_bins + (size_t)r * NB;
    for (int j = lane; j < NB; j += 32) {
      // u: stratified (linspace(0, 1 - 1/NB, NB) + rand / NB) or bin centres
      float u = A.u_base[j];
      if (A.u_rand) u = __fadd_rn(u, __fdiv_rn(A.u_rand[(size_t)r * A.u_stride + (A.u_stride > 1 ? j : 0)], (float)NB));
      else u = __fadd_rn(u, (float)(1.0 / (2.0 * (double)NB)));
      // searchsorted(cdf, u, side="right"): number of entries <= u
      int lo = 0, hi = S + 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cdf[mid] <= u) lo = mid + 1;
        else hi = mid;
      }
      const int below = min(max(lo - 1, 0), S), above = min(max(lo, 0), S);
      const float c0v = cdf[below], c1v = cdf[above];
      float t = (u - c0v) / (c1v - c0v);
      if (t != t) t = 0.f;  // nan_to_num(., 0); +-inf are clipped below
      t = fminf(fmaxf(t, 0.f), 1.f);
      const float b0 = eb[below], b1 = eb[above];
      const float nb = b0 + t * (b1 - b0);
      out_bins[j] = nb;
      const float e = lindisp_inv(nb * far_s + (1.0f - nb) * near_s);
      if (j < A.num_samples) A.starts[(size_t)r * A.num_samples + j] = e;
      if (j > 0) A.ends[(size_t)r * A.num_samples + j - 1] = e;
    }
    __syncwarp();
  }
}

// ---- interlevel loss ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * kWarpsPerBlock) interlevel_loss_kernel(KInterlevel A) {
  __shared__ float s_cy[kWarpsPerBlock][kMaxPdfBins + 1];
  __shared__ float s_dcy[kWarpsPerBlock][kMaxPdfBins + 1];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* cy = s_cy[wib];
  float* dcy = s_dcy[wib];
  const int Sc = A.Sc, Sp = A.Sp;
  float loss_part = 0.f;
  for (int r = blockIdx.x * kWarpsPerBlock + wib; r < A.R; r += gridDim.x * kWarpsPerBlock) {
    const float* c = A.c + (size_t)r * (Sc + 1);
    const float* w = A.w + (size_t)r * Sc;
    const float* cp = A.cp + (size_t)r * (Sp + 1);
    const float* wp = A.wp + (size_t)r * Sp;
    // cy = [0, cumsum(wp)]
    if (lane == 0) cy[0] = 0.f;
    warp_cumsum(Sp, lane, [&](int i) { return wp[i]; }, [&](int i, float c) { cy[i + 1] = c; });
    for (int i = lane; i <= Sp; i += 32) dcy[i] = 0.f;
    __syncwarp();
    for (int i = lane; i < Sc; i += 32) {
      const float t0s = c[i], t0e = c[i + 1];
      // idx_lo = searchsorted(cp[:-1], t0s, right) - 1 ; idx_hi = searchsorted(cp[1:], t0e, right); clamp to [0, Sp-1]
      int lo = 0, hi = Sp;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cp[mid] <= t0s) lo = mid + 1;
        else hi = mid;
      }
      const int idx_lo = min(max(lo - 1, 0), Sp - 1);
      lo = 0;
      hi = Sp;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cp[mid + 1] <= t0e) lo = mid + 1;
        else hi = mid;
      }
      const int idx_hi = min(max(lo, 0), Sp - 1);
      const float w_outer = cy[idx_hi + 1] - cy[idx_lo];
      const float wi = w[i];
      const float diff = fmaxf(wi - w_outer, 0.f);
      loss_part += diff * diff / (wi + 1.0e-7f);
      if (A.d_wp && diff > 0.f) {
        const float g = -2.0f * diff / (wi + 1.0e-7f) * A.scale;
        atomicAdd(&dcy[idx_hi + 1], g);
        atomicAdd(&dcy[idx_lo], -g);
      }
    }
    __syncwarp();
    if (A.d_wp) {
      // d wp[k] = sum_{m >= k+1} dcy[m]  (suffix sum)
      float* dwp = A.d_wp + (size_t)r * Sp;
      float tot = 0.f;
      for (int i = lane; i <= Sp; i += 32) tot += dcy[i];
      tot = warp_sum(tot);
      // suffix over m >= i+1  = tot - prefix(i)
      warp_cumsum(Sp + 1, lane, [&](int i) { return dcy[i]; }, [&](int i, float c) {
        if (i < Sp) dwp[i] = tot - c;
      });
    }
    __syncwarp();
  }
  loss_part = warp_sum(loss_part);
  if (lane == 0 && loss_part != 0.f) atomicAdd(A.loss, loss_part * A.scale);
}

}  // namespace

int launch_proposal_weights_forward(const KDensity& D, const KRays& Rr, float* density, float* weights, cudaStream_t st) {
  if (Rr.R == 0) return FNR_OK;
  const int grid = grid_for(Rr.R, kWarpsPerBlock, sm_count() * 16);
  proposal_weights_forward_kernel<<<grid, 32 * kWarpsPerBlock, 0, st>>>(D, Rr, density, weights);
  return check_launch("proposal_weights_forward_kernel");
}

int launch_proposal_weights_backward(const KDensity& D, const KDensity& G, const KRays& Rr, const float* density, const float* weights,
                                     const float* d_weights, cudaStream_t st) {
  if (Rr.R == 0) return FNR_OK;
  const int grid = grid_for(Rr.R, kWarpsPerBlock, sm_count() * 4);
  proposal_weights_backward_kernel<<<grid, 32 * kWarpsPerBlock, 0, st>>>(D, G, Rr, density, weights, d_weights);
  return check_launch("proposal_weights_backward_kernel");
}

int launch_pdf_sample(const KPdf& A, cudaStream_t st) {
  if (A.R == 0) return FNR_OK;
  pdf_sample_kernel<<<grid_for(A.R, kWarpsPerBlock, sm_count() * 16), 32 * kWarpsPerBlock, 0, st>>>(A);
  return check_launch("pdf_sample_kernel");
}

int launch_interlevel_loss(const KInterlevel& A, cudaStream_t st) {
  if (A.R == 0) return FNR_OK;
  interlevel_loss_kernel<<<grid_for(A.R, kWarpsPerBlock, sm_count() * 16), 32 * kWarpsPerBlock, 0, st>>>(A);
  return check_launch("interlevel_loss_kernel");
}

int proposal_limits(int* max_levels, int* hidden, int* max_bins) {
  *max_levels = kMaxLevels;
  *hidden = kHidden;
  *max_bins = kMaxPdfBins;
  return 0;
}

}  // namespace fnr
