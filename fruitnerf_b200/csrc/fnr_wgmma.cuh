// Hopper (sm_90a) warpgroup MMA layer: the MLP layers of the tensor-core field forward and backward (fnr_simt.cu,
// Layers<C, true>): y = W x + b, dx = W^T dy and dW = dY^T X of a 128-point tile.
//
// One CTA of 128 threads = one warpgroup = one tile of 128 sample points, thread t owning point t.  A layer
// y = W x + b is one block-wide step: every thread writes its row x[K] into shared memory as a bf16 hi/lo split
// (x ~= hi + lo, 16 mantissa bits), the weights W[N][K] are split the same way, and the warpgroup runs
// D[128, N] = Xhi Whi^T + Xlo Whi^T + Xhi Wlo^T + Xlo Wlo^T with fp32 accumulation (wgmma m64nNk16, two M halves);
// the accumulator fragments go back to shared memory in fp32 and every thread reads its row.  Relative error of a
// product ~2^-17 (the rounding of the lo halves), fp32-class for the parity bar of the tests.
//
// Operand layout (no swizzle, K-major core matrices of 8 rows x 16 bytes): element (row, k) of a ROWS x KP tile is at
//     (k / 8) * (ROWS * 16) + row * 16 + (k % 8) * 2
// so the descriptor's leading byte offset (between the two K core matrices of one k16 step) is ROWS * 16 and its
// stride byte offset (between 8-row groups) is 128.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

// Diagnostic build of the backward (-DFNR_BWD_PHASE_TIMERS, tools/bench_backward.py --phases; never set by the normal
// build): FNR_PHASE(i) closes phase i of the current tile.  Every thread of the CTA calls it; after a barrier, thread 0
// adds the clock64() cycles since the previous mark to the CTA's counter of phase i.
namespace fnr {
enum BwdPhase { kPhLoad, kPhRecompute, kPhDx, kPhDw, kPhDwFlush, kPhScatter, kBwdPhases };
#ifdef FNR_BWD_PHASE_TIMERS
namespace phase {
__shared__ unsigned long long cycles[kBwdPhases];
__shared__ long long last;
__device__ __forceinline__ void mark(int i) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const long long now = clock64();
    cycles[i] += (unsigned long long)(now - last);
    last = now;
  }
}
}  // namespace phase
#define FNR_PHASE(i) ::fnr::phase::mark(i)
#else
#define FNR_PHASE(i) ((void)0)
#endif
}  // namespace fnr

namespace fnr {
namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// sm_90 shared-memory matrix descriptor: start, leading / stride byte offsets in 16-byte units, no swizzle.
__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}

__device__ __forceinline__ void fence_operands() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// generic-proxy shared-memory stores -> visible to the async proxy that wgmma reads operands through
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// D[64, N] (+)= A[64, 16] B[N, 16]^T, bf16 operands from shared memory, fp32 accumulators in registers.
template <int N>
__device__ __forceinline__ void mma_m64k16(float (&d)[N / 2], uint64_t a, uint64_t b, int scale_d);
template <>
__device__ __forceinline__ void mma_m64k16<16>(float (&d)[8], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void mma_m64k16<32>(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void mma_m64k16<64>(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void mma_m64k16<128>(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}

__device__ __forceinline__ void split_store(uint8_t* hi, uint8_t* lo, int off, float x) {
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  *reinterpret_cast<__nv_bfloat16*>(hi + off) = h;
  *reinterpret_cast<__nv_bfloat16*>(lo + off) = __float2bfloat16_rn(x - __bfloat162float(h));
}

// hi / lo split of 8 consecutive k of one row: one core-matrix row, one 16-byte store into each half.
__device__ __forceinline__ void split_store8(uint8_t* hi, uint8_t* lo, int off, const float (&x)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 hv = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
    const float2 hf = __bfloat1622float2(hv);
    const __nv_bfloat162 lv = __floats2bfloat162_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hv);
    l[i] = *reinterpret_cast<const uint32_t*>(&lv);
  }
  *reinterpret_cast<uint4*>(hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

constexpr int pad16(int k) { return (k + 15) / 16 * 16; }
constexpr int padn(int n) { return n <= 16 ? 16 : n <= 32 ? 32 : n <= 64 ? 64 : 128; }

// Shared memory of one layer step: X tile (hi | lo), W tile (hi | lo), fp32 result rows.
template <int KMAX, int NMAX>
struct Smem {
  static constexpr int kX = 2 * 128 * pad16(KMAX) * 2;
  static constexpr int kW = 2 * padn(NMAX) * pad16(KMAX) * 2;
  static constexpr int kYStride = padn(NMAX) + 4;  // floats per result row
  static constexpr int kBytes = kX + kW + 128 * kYStride * 4;
};

// Per-thread-row GEMM y[NO] = sum_r x[r] * getw(no, r) for the point of this thread (getw: fp32 weight of output no,
// reduction index r); every thread of the CTA (one warpgroup) must call it.
template <int KMAX, int NMAX, int R, int NO, class GetW>
__device__ __forceinline__ void rowgemm(uint8_t* smem, const float (&x)[R], float (&y)[NO], GetW getw) {
  constexpr int KP = pad16(R), NP = padn(NO);
  static_assert(KP <= pad16(KMAX) && NP <= padn(NMAX), "layer larger than the shared-memory plan");
  using S = Smem<KMAX, NMAX>;
  uint8_t* xhi = smem;
  uint8_t* xlo = smem + 128 * KP * 2;
  uint8_t* whi = smem + S::kX;
  uint8_t* wlo = whi + NP * KP * 2;
  float* ys = reinterpret_cast<float*>(smem + S::kX + S::kW);
  const int t = threadIdx.x;
  __syncthreads();  // the previous step's readers are done with every buffer
#pragma unroll
  for (int kc = 0; kc < KP / 8; ++kc) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 8 * kc + j < R ? x[8 * kc + j < R ? 8 * kc + j : 0] : 0.f;
    split_store8(xhi, xlo, kc * (128 * 16) + t * 16, v);
  }
  // weight tile in (row, 8-k chunk) units, consecutive threads on consecutive rows of one chunk column
  constexpr int kChunks = NP * KP / 8;
#pragma unroll 1
  for (int it = 0; it < (kChunks + 127) / 128; ++it) {
    const int i = t + 128 * it;
    if (kChunks % 128 != 0 && i >= kChunks) break;
    const int n = i % NP, kc = i / NP;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (n < NO && 8 * kc + j < R) ? getw(n, 8 * kc + j) : 0.f;
    split_store8(whi, wlo, kc * (NP * 16) + n * 16, v);
  }
  fence_proxy_async();
  __syncthreads();
  const uint32_t ax = smem_u32(xhi), aw = smem_u32(whi);
  constexpr uint32_t XLO = 128 * KP * 2, WLO = NP * KP * 2;
  const int warp = t >> 5, lane = t & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float d[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) d[i] = 0.f;
    fence_operands();
#pragma unroll
    for (int ks = 0; ks < KP / 16; ++ks) {
      const uint32_t xa = ax + ks * 2 * (128 * 16) + h * 64 * 16, wa = aw + ks * 2 * (NP * 16);
      const uint64_t dxh = desc(xa, 128 * 16, 128), dxl = desc(xa + XLO, 128 * 16, 128);
      const uint64_t dwh = desc(wa, NP * 16, 128), dwl = desc(wa + WLO, NP * 16, 128);
      mma_m64k16<NP>(d, dxh, dwh, ks > 0);
      mma_m64k16<NP>(d, dxl, dwh, 1);
      mma_m64k16<NP>(d, dxh, dwl, 1);
      mma_m64k16<NP>(d, dxl, dwl, 1);
    }
    commit();
    wait_all();
    // fragment (i, j): row 16 * warp + lane / 4 (+8 for j >= 2), column 8 * i + 2 * (lane % 4) + (j & 1)
    const int r0 = h * 64 + 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < NP / 8; ++i) {
      *reinterpret_cast<float2*>(ys + r0 * S::kYStride + 8 * i + c0) = make_float2(d[4 * i], d[4 * i + 1]);
      *reinterpret_cast<float2*>(ys + (r0 + 8) * S::kYStride + 8 * i + c0) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
  }
  __syncthreads();
  // row t, 16-byte aligned (kYStride is a multiple of 4)
#pragma unroll
  for (int n = 0; n < NO / 4 * 4; n += 4) {
    const float4 v = *reinterpret_cast<const float4*>(ys + t * S::kYStride + n);
    y[n] = v.x;
    y[n + 1] = v.y;
    y[n + 2] = v.z;
    y[n + 3] = v.w;
  }
#pragma unroll
  for (int n = NO / 4 * 4; n < NO; ++n) y[n] = ys[t * S::kYStride + n];
}

// y[N] = W x + b (optionally ReLU), W in torch layout [N][K].
template <int KMAX, int NMAX, int K, int N, bool RELU>
__device__ __forceinline__ void linear(uint8_t* smem, const float* __restrict__ W, const float* __restrict__ b, const float (&x)[K],
                                       float (&y)[N]) {
  rowgemm<KMAX, NMAX, K, N>(smem, x, y, [&](int n, int k) { return __ldg(W + (size_t)n * K + k); });
#pragma unroll
  for (int n = 0; n < N; ++n) {
    const float v = y[n] + __ldg(b + n);
    y[n] = RELU ? fmaxf(v, 0.f) : v;
  }
}

// Input gradient dx[K] = W^T dy for W [N][K] (the same GEMM with the weight read transposed).
template <int KMAX, int NMAX, int K, int N>
__device__ __forceinline__ void linear_dx(uint8_t* smem, const float* __restrict__ W, const float (&dy)[N], float (&dx)[K]) {
  rowgemm<KMAX, NMAX, N, K>(smem, dy, dx, [&](int k, int n) { return __ldg(W + (size_t)n * K + k); });
}

// Shared memory of one weight-gradient step: dY^T tile [MP x 128 points] (hi | lo), X^T tile [KP x 128] (hi | lo), fp32 dY rows.
template <int K, int N>
struct DwSmem {
  static constexpr int MP = N <= 64 ? 64 : 128, KP = padn(K), YS = MP + 4;
  static constexpr int kA = 2 * MP * 128 * 2, kB = 2 * KP * 128 * 2;
  static constexpr int kBytes = kA + kB + 128 * YS * 4;
};

// Weight gradient of the CTA's 128-point tile, gW[N][K] += dY^T X and gb[N] += column sums of dY, both operands read
// K-major over the points (the reduction dimension); accumulated in warpgroup registers and added to the global gradient once
// per tile.  Every thread of the CTA must call it.
template <int K, int N>
__device__ __forceinline__ void weight_grad(uint8_t* smem, const float (&x)[K], const float (&dy)[N], float* __restrict__ gW,
                                            float* __restrict__ gb) {
  using S = DwSmem<K, N>;
  constexpr int MP = S::MP, KP = S::KP;
  uint8_t* ahi = smem;
  uint8_t* alo = smem + MP * 128 * 2;
  uint8_t* bhi = smem + S::kA;
  uint8_t* blo = bhi + KP * 128 * 2;
  float* ys = reinterpret_cast<float*>(smem + S::kA + S::kB);
  const int t = threadIdx.x;
  __syncthreads();
  // point t is reduction index t: element (row, t) at (t / 8) * (ROWS * 16) + row * 16 + (t % 8) * 2
  const int pt = (t >> 3) * 16, pl = (t & 7) * 2;
#pragma unroll
  for (int n = 0; n < MP; ++n) {
    const float v = n < N ? dy[n < N ? n : 0] : 0.f;
    split_store(ahi, alo, pt * MP + n * 16 + pl, v);
    if (n < N) ys[t * S::YS + n] = v;
  }
#pragma unroll
  for (int k = 0; k < KP; ++k) split_store(bhi, blo, pt * KP + k * 16 + pl, k < K ? x[k < K ? k : 0] : 0.f);
  fence_proxy_async();
  __syncthreads();
  const uint32_t aa = smem_u32(ahi), ab = smem_u32(bhi);
  constexpr uint32_t ALO = MP * 128 * 2, BLO = KP * 128 * 2;
  const int warp = t >> 5, lane = t & 31;
#pragma unroll
  for (int h = 0; h < MP / 64; ++h) {
    float d[KP / 2];
#pragma unroll
    for (int i = 0; i < KP / 2; ++i) d[i] = 0.f;
    fence_operands();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t xa = aa + ks * 2 * (MP * 16) + h * 64 * 16, wa = ab + ks * 2 * (KP * 16);
      const uint64_t dah = desc(xa, MP * 16, 128), dal = desc(xa + ALO, MP * 16, 128);
      const uint64_t dbh = desc(wa, KP * 16, 128), dbl = desc(wa + BLO, KP * 16, 128);
      mma_m64k16<KP>(d, dah, dbh, ks > 0);
      mma_m64k16<KP>(d, dal, dbh, 1);
      mma_m64k16<KP>(d, dah, dbl, 1);
      mma_m64k16<KP>(d, dal, dbl, 1);
    }
    commit();
    wait_all();
    FNR_PHASE(kPhDw);
    const int n0 = h * 64 + 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < KP / 8; ++i) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + (j >= 2 ? 8 : 0), k = 8 * i + c0 + (j & 1);
        if (n < N && k < K && d[4 * i + j] != 0.f) atomicAdd(gW + (size_t)n * K + k, d[4 * i + j]);
      }
    }
  }
  __syncthreads();
  for (int n = t; n < N; n += 128) {  // bias: column sums of dY in fp32
    float sum = 0.f;
    for (int p = 0; p < 128; ++p) sum += ys[p * S::YS + n];
    if (sum != 0.f) atomicAdd(gb + n, sum);
  }
  FNR_PHASE(kPhDwFlush);
}

}  // namespace wg
}  // namespace fnr
