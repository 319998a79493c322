// Fused multi-tensor Adam / RAdam step over the flat parameter / gradient buffers (the optimiser half of
// a training iteration: nerfstudio Optimizers.optimizer_step_all with the optimisers of
// fruit_nerf/fruit_nerf_config.py:47-56, 90-103).  One launch updates every tensor of a param group;
// hyper-parameters (learning rate, bias corrections) live in DEVICE memory so the launch can sit inside a
// captured CUDA graph while the schedule advances.  HBM-bound: 16 B read + 12 B written per element.
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;

// hyper[]: 0 lr, 1 beta1, 2 beta2, 3 eps, 4 bias_correction1, 5 bias_correction2, 6 radam rectification
// (< 0: variance not tractable yet -> un-adapted step), 7 grad_scale (e.g. 1/world_size; 1 = none)
template <bool kRAdam>
__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, const float* __restrict__ h) {
  const float lr = h[0], b1 = h[1], b2 = h[2], eps = h[3], bc1 = h[4], bc2 = h[5], rect = h[6];
  g *= h[7];
  m = fmaf(b1, m, (1.0f - b1) * g);        // exp_avg.lerp_(grad, 1 - beta1)
  v = fmaf(b2, v, (1.0f - b2) * g * g);    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
  if (kRAdam) {
    const float mh = m / bc1;
    if (rect >= 0.f)
      p -= mh * lr * (sqrtf(bc2) / (sqrtf(v) + eps)) * rect;
    else
      p -= mh * lr;
  } else {
    const float denom = sqrtf(v) / sqrtf(bc2) + eps;
    p -= (lr / bc1) * (m / denom);
  }
}

template <bool kRAdam>
__global__ void __launch_bounds__(kThreads) adam_kernel(KAdam A, const float* __restrict__ hyper) {
  __shared__ float h[8];
  if (threadIdx.x < 8) h[threadIdx.x] = hyper[threadIdx.x];
  __syncthreads();
  for (int t = 0; t < A.count; ++t) {
    const KAdamTensor T = A.t[t];
    const long long n4 = T.vec4 ? T.n / 4 : 0;
    float4* p4 = reinterpret_cast<float4*>(T.param);
    const float4* g4 = reinterpret_cast<const float4*>(T.grad);
    float4* m4 = reinterpret_cast<float4*>(T.exp_avg);
    float4* v4 = reinterpret_cast<float4*>(T.exp_avg_sq);
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n4; i += (long long)gridDim.x * kThreads) {
      float4 p = p4[i], m = m4[i], v = v4[i];
      const float4 g = g4[i];
      adam_update<kRAdam>(p.x, g.x, m.x, v.x, h);
      adam_update<kRAdam>(p.y, g.y, m.y, v.y, h);
      adam_update<kRAdam>(p.z, g.z, m.z, v.z, h);
      adam_update<kRAdam>(p.w, g.w, m.w, v.w, h);
      p4[i] = p;
      m4[i] = m;
      v4[i] = v;
    }
    for (long long i = 4 * n4 + (long long)blockIdx.x * kThreads + threadIdx.x; i < T.n; i += (long long)gridDim.x * kThreads) {
      float p = T.param[i], m = T.exp_avg[i], v = T.exp_avg_sq[i];
      adam_update<kRAdam>(p, T.grad[i], m, v, h);
      T.param[i] = p;
      T.exp_avg[i] = m;
      T.exp_avg_sq[i] = v;
    }
  }
}

}  // namespace

int launch_adam(const KAdam& A, int radam, const float* hyper, cudaStream_t st) {
  long long total = 0;
  for (int t = 0; t < A.count; ++t) total += A.t[t].n;
  if (total == 0) return FNR_OK;
  const int blocks = grid_for(total / 4, kThreads, sm_count() * 8);
  if (radam)
    adam_kernel<true><<<blocks, kThreads, 0, st>>>(A, hyper);
  else
    adam_kernel<false><<<blocks, kThreads, 0, st>>>(A, hyper);
  return check_launch("adam_kernel");
}

}  // namespace fnr
