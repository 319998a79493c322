// Hopper (sm_90a) warpgroup MMA layer: the MLP layers of the tensor-core field forward and backward (fnr_simt.cu,
// Layers<C, true> and ResidentLayers): y = W x + b, dx = W^T dy and dW = dY^T X of a 128-point tile.
//
// One warpgroup (128 threads) = one tile of 128 sample points, thread t of the warpgroup owning point t.  A layer
// y = W x + b is one warpgroup-wide step: every thread writes its row x[K] into shared memory as a bf16 hi/lo split
// (x ~= hi + lo, 16 mantissa bits), the weights W[N][K] are split the same way, and the warpgroup runs
// D[128, N] = Xhi Whi^T + Xlo Whi^T + Xhi Wlo^T + Xlo Wlo^T with fp32 accumulation (wgmma m64nNk16, two M halves);
// the accumulator fragments go back to shared memory in fp32 and every thread reads its row.  Relative error of a
// product ~2^-17 (the rounding of the lo halves), fp32-class for the parity bar of the tests.  The small family's forward,
// export and backward (CTAs of several warpgroups) split their weights once per CTA into a resident image, and the backward
// accumulates dW / db in shared memory; the big family's kernels (one warpgroup per CTA) stage the weight tile from global
// memory at every step.  Where a layer's only consumer is the next layer (resident_chain), its fragments are stored
// straight into the next layer's operand tile instead of going through rows.
//
// Operand layout (no swizzle, core matrices of 8 rows x 16 bytes).  K-major: element (row, k) of a ROWS x KP tile is at
//     (k / 8) * (ROWS * 16) + row * 16 + (k % 8) * 2
// MN-major (read with the wgmma transpose bit): element (row, k) is at (row / 8) * MN_STRIDE + k * 16 + (row % 8) * 2.
// In both, a descriptor's leading byte offset is the stride between core matrices along K and its stride byte offset
// the stride between core matrices along M / N (K-major: ROWS * 16 and 128; MN-major: 128 and MN_STRIDE).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace fnr {
namespace wg {
// Index of the thread in its warpgroup, the warpgroup in the CTA, and the warpgroup's named barrier (id 1 + warpgroup;
// id 0 is __syncthreads).  A CTA of one warpgroup sees threadIdx.x and a barrier over the whole CTA.
__device__ __forceinline__ int tid() { return threadIdx.x & 127; }
__device__ __forceinline__ int group() { return threadIdx.x >> 7; }
__device__ __forceinline__ void sync() { asm volatile("bar.sync %0, 128;" ::"r"(1 + group()) : "memory"); }
}  // namespace wg

// Diagnostic build of the backward (-DFNR_BWD_PHASE_TIMERS, tools/bench_backward.py --phases; never set by the normal
// build): FNR_PHASE(i) closes phase i of the current tile.  Every thread of the warpgroup calls it; after the warpgroup's
// barrier, its thread 0 adds the clock64() cycles since the previous mark to the warpgroup's counter of phase i.
enum BwdPhase { kPhLoad, kPhRecompute, kPhDx, kPhDw, kPhDwFlush, kPhScatter, kBwdPhases };
#ifdef FNR_BWD_PHASE_TIMERS
namespace phase {
__shared__ unsigned long long cycles[2][kBwdPhases];
__shared__ long long last[2];
__device__ __forceinline__ void mark(int i) {
  wg::sync();
  if (wg::tid() == 0) {
    const long long now = clock64();
    cycles[wg::group()][i] += (unsigned long long)(now - last[wg::group()]);
    last[wg::group()] = now;
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

// mbarriers in shared memory (a ring between warpgroups of a CTA): init by one thread, then a CTA barrier before use;
// arrive has release and a completed wait acquire semantics at CTA scope, so the generic-proxy stores before an arrive
// are visible to the loads after the wait that sees its phase complete.
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Waits until the phase with parity `parity` of the barrier has completed.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred done;\n"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 done, [%0], %1;\n\t"
      "@!done bra WAIT_%=;\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// The registers per thread of the calling warpgroup (warpgroup-uniform; the CTA's sum must stay within what it was
// launched with).
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// D[64, N] (+)= A[64, 16] B[N, 16]^T, bf16 operands from shared memory, fp32 accumulators in registers.  TA / TB: the
// operand is MN-major (the transpose bit).
template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void mma_m64k16(float (&d)[N / 2], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (N == 16) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
  } else if constexpr (N == 32) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
  } else if constexpr (N == 64) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
  } else {
    static_assert(N == 128, "wgmma tile width");
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB));
  }
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

// hi / lo split of values [8 c, 8 c + 8) of a register vector (zero past R) into one core-matrix row.
template <int R>
__device__ __forceinline__ void split_store_chunk(uint8_t* hi, uint8_t* lo, int off, const float (&x)[R], int c) {
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 8 * c + j < R ? x[8 * c + j < R ? 8 * c + j : 0] : 0.f;
  split_store8(hi, lo, off, v);
}

constexpr int pad16(int k) { return (k + 15) / 16 * 16; }
constexpr int padn(int n) { return n <= 16 ? 16 : n <= 32 ? 32 : n <= 64 ? 64 : 128; }

// Shared memory of one staged layer step: X tile (hi | lo), W tile (hi | lo), fp32 result rows.
template <int KMAX, int NMAX>
struct Smem {
  static constexpr int kX = 2 * 128 * pad16(KMAX) * 2;
  static constexpr int kW = 2 * padn(NMAX) * pad16(KMAX) * 2;
  static constexpr int kYStride = padn(NMAX) + 4;  // floats per result row
  static constexpr int kBytes = kX + kW + 128 * kYStride * 4;
};

// Shared memory of one resident layer step (ResidentLayers): the X tile, with the fp32 result rows stored over it as
// they are produced.  Result element (row, c) is at float (c / 4) * 512 + row * 4 + c % 4: column group c / 4 takes the
// 2 KiB of one 8-k chunk of the tile (hi or lo), and M half h writes rows [64 h, 64 h + 64), the 1 KiB of each chunk
// that its MMAs have just consumed.  The fragment stores and the row reads are free of bank conflicts.
constexpr int kResidentStepBytes = 2 * 128 * 64 * 2;
constexpr int kRowsGroupStride = 512;

// B operand of a layer step: W [NP outputs] x [KP reduction], hi at `hi`, lo `lo` bytes further; lbo / sbo as in the
// descriptor, `kstep` bytes between k16 steps.
struct BOperand {
  uint32_t hi, lo, lbo, sbo, kstep;
};

// The MMA sequence of a layer step and its write-back: D[128, NP] = X W^T over the X tile at `ax` (K-major, lo `xlo`
// bytes further) as hi.hi, lo.hi, hi.lo, lo.lo per k16 step, M half by M half, each half's fragments stored as fp32 at
// ys + row * row_stride + (c / 4) * group_stride + c % 4.  ALIAS: ys lies over the X tile, so the warpgroup waits for
// all of a half's MMAs before any of its rows is stored.  Every thread of the warpgroup must call it.
template <int KP, int NP, int TB, bool ALIAS>
__device__ __forceinline__ void layer_mma(uint32_t ax, uint32_t xlo, const BOperand& w, float* ys, int row_stride, int group_stride) {
  const int t = tid(), warp = t >> 5, lane = t & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float d[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) d[i] = 0.f;
    fence_operands();
#pragma unroll
    for (int ks = 0; ks < KP / 16; ++ks) {
      const uint32_t xa = ax + ks * 2 * (128 * 16) + h * 64 * 16, wa = w.hi + ks * w.kstep;
      const uint64_t dxh = desc(xa, 128 * 16, 128), dxl = desc(xa + xlo, 128 * 16, 128);
      const uint64_t dwh = desc(wa, w.lbo, w.sbo), dwl = desc(wa + w.lo, w.lbo, w.sbo);
      mma_m64k16<NP, 0, TB>(d, dxh, dwh, ks > 0);
      mma_m64k16<NP, 0, TB>(d, dxl, dwh, 1);
      mma_m64k16<NP, 0, TB>(d, dxh, dwl, 1);
      mma_m64k16<NP, 0, TB>(d, dxl, dwl, 1);
    }
    commit();
    wait_all();
    if (ALIAS) sync();
    // fragment (i, j): row 16 * warp + lane / 4 (+8 for j >= 2), column 8 * i + 2 * (lane % 4) + (j & 1)
    const int r0 = h * 64 + 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < NP / 8; ++i) {
      float* y = ys + (2 * i + (c0 >> 2)) * group_stride + (c0 & 3);
      *reinterpret_cast<float2*>(y + r0 * row_stride) = make_float2(d[4 * i], d[4 * i + 1]);
      *reinterpret_cast<float2*>(y + (r0 + 8) * row_stride) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
  }
}

// This thread's result row of layer_mma (16-byte aligned groups of 4), after a warpgroup barrier.
template <int NO>
__device__ __forceinline__ void read_row(const float* ys, int row_stride, int group_stride, float (&y)[NO]) {
  const float* r = ys + tid() * row_stride;
#pragma unroll
  for (int n = 0; n < NO / 4 * 4; n += 4) {
    const float4 v = *reinterpret_cast<const float4*>(r + (n / 4) * group_stride);
    y[n] = v.x;
    y[n + 1] = v.y;
    y[n + 2] = v.z;
    y[n + 3] = v.w;
  }
#pragma unroll
  for (int n = NO / 4 * 4; n < NO; ++n) y[n] = r[(n / 4) * group_stride + n % 4];
}

// Per-thread-row GEMM y[NO] = sum_r x[r] * getw(no, r) for the point of this thread (getw: fp32 weight of output no,
// reduction index r), with the weight tile staged from getw; every thread of the CTA (one warpgroup) must call it.
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
  const int t = tid();
  __syncthreads();  // the previous step's readers are done with every buffer
#pragma unroll
  for (int kc = 0; kc < KP / 8; ++kc) split_store_chunk(xhi, xlo, kc * (128 * 16) + t * 16, x, kc);
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
  const BOperand w{smem_u32(whi), (uint32_t)(NP * KP * 2), NP * 16, 128, 2 * NP * 16};
  layer_mma<KP, NP, 0, false>(smem_u32(xhi), 128 * KP * 2, w, ys, S::kYStride, 4);
  __syncthreads();
  read_row<NO>(ys, S::kYStride, 4, y);
}

// The MMA sequence of layer_mma with both M halves' chains issued back to back into d[0] and d[1], then one wait and one
// warpgroup barrier: after it, every read of the X tile is done and the tile may be overwritten.  The fragments stay in
// registers, in layer_mma's fragment order.  Every thread of the warpgroup must call it.
template <int KP, int NP, int TB>
__device__ __forceinline__ void layer_mma_frag(uint32_t ax, uint32_t xlo, const BOperand& w, float (&d)[2][NP / 2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) d[h][i] = 0.f;
  fence_operands();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int ks = 0; ks < KP / 16; ++ks) {
      const uint32_t xa = ax + ks * 2 * (128 * 16) + h * 64 * 16, wa = w.hi + ks * w.kstep;
      const uint64_t dxh = desc(xa, 128 * 16, 128), dxl = desc(xa + xlo, 128 * 16, 128);
      const uint64_t dwh = desc(wa, w.lbo, w.sbo), dwl = desc(wa + w.lo, w.lbo, w.sbo);
      mma_m64k16<NP, 0, TB>(d[h], dxh, dwh, ks > 0);
      mma_m64k16<NP, 0, TB>(d[h], dxl, dwh, 1);
      mma_m64k16<NP, 0, TB>(d[h], dxh, dwl, 1);
      mma_m64k16<NP, 0, TB>(d[h], dxl, dwl, 1);
    }
  }
  commit();
  wait_all();
  sync();
}

// stmatrix of four 8 x 8 b16 matrices: lane l gives the address of row l % 8 of matrix l / 8 (16 contiguous bytes), and
// register m holds the lane's elements (row lane / 4, columns 2 (lane % 4) and + 1) of matrix m, the first in the low half.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

// The fragments of layer_mma_frag (NP columns) as the next layer's K-major A tile of K = NP at `tile` (lo 128 * NP * 2 bytes
// further), split hi / lo per element as split_store8 splits a row, so the bytes are the ones split_store_chunk would write
// from the same values.  An m64nN accumulator fragment has the layout of stmatrix.m8n8: the warp's rows 16 warp + [0, 8) and
// + [8, 16) of k chunks i and i + 1 are four core matrices, one x4 store into hi and one into lo.
template <int NP>
__device__ __forceinline__ void store_a_tile(uint32_t tile, const float (&d)[2][NP / 2]) {
  const int t = tid(), warp = t >> 5, lane = t & 31, m = lane >> 3;
  constexpr uint32_t LO = 128 * NP * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    // matrix m: k chunk i + m / 2, rows + 8 (m % 2); its fragment values are d[h][4 (i + m / 2) + 2 (m % 2) + {0, 1}]
    const uint32_t row = h * 64 + 16 * warp + 8 * (m & 1) + (lane & 7);
#pragma unroll
    for (int i = 0; i < NP / 8; i += 2) {
      uint32_t hr[4], lr[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float v0 = d[h][4 * (i + q / 2) + 2 * (q & 1)], v1 = d[h][4 * (i + q / 2) + 2 * (q & 1) + 1];
        const __nv_bfloat162 hv = __floats2bfloat162_rn(v0, v1);
        const float2 hf = __bfloat1622float2(hv);
        const __nv_bfloat162 lv = __floats2bfloat162_rn(v0 - hf.x, v1 - hf.y);
        hr[q] = *reinterpret_cast<const uint32_t*>(&hv);
        lr[q] = *reinterpret_cast<const uint32_t*>(&lv);
      }
      const uint32_t a = tile + (i + (m >> 1)) * (128 * 16) + row * 16;
      stmatrix_x4(a, hr);
      stmatrix_x4(a + LO, lr);
    }
  }
}

// The resident image's B operand of slot image `img` (W [NPF][KPF] K-major): read K-major for y = W x, MN-major through
// the transpose bit for y = W^T x.
template <int NPF, int KPF, bool TRANS>
__device__ __forceinline__ BOperand image_operand(const uint8_t* img) {
  const uint32_t iw = smem_u32(img), lo = NPF * KPF * 2;
  return TRANS ? BOperand{iw, lo, 128, NPF * 16, 2 * 128} : BOperand{iw, lo, NPF * 16, 128, 2 * NPF * 16};
}

// The row tile of a resident step: every thread splits its row x[R] into the warpgroup's K-major X tile, after the
// previous step's readers are done with it.
template <int R>
__device__ __forceinline__ void stage_rows(uint8_t* smem, const float (&x)[R]) {
  constexpr int KP = pad16(R);
  const int t = tid();
  sync();  // the previous step's readers are done with the tile
#pragma unroll
  for (int kc = 0; kc < KP / 8; ++kc) split_store_chunk(smem, smem + 128 * KP * 2, kc * (128 * 16) + t * 16, x, kc);
  fence_proxy_async();
  sync();
}

// y = W^T x (dx) on the row tile of x[R] already staged in smem (stage_rows' bytes), with the weights from a resident
// split image (W [NPF][KPF] K-major, as rowgemm stages it) read MN-major through the transpose bit; the result rows are
// stored over the tile.  smem is the warpgroup's kResidentStepBytes.
template <int NPF, int KPF, int R, int NO>
__device__ __forceinline__ void resident_rowgemm_t_staged(uint8_t* smem, const uint8_t* img, float (&y)[NO]) {
  constexpr int KP = pad16(R), NP = padn(NO);
  static_assert(KP <= NPF && NP <= KPF, "layer outside the resident image");
  static_assert(2 * 128 * KP * 2 <= kResidentStepBytes && NP * 128 * 4 <= kResidentStepBytes, "resident step plan");
  float* ys = reinterpret_cast<float*>(smem);
  layer_mma<KP, NP, 1, true>(smem_u32(smem), 128 * KP * 2, image_operand<NPF, KPF, true>(img), ys, 4, kRowsGroupStride);
  sync();
  read_row<NO>(ys, 4, kRowsGroupStride, y);
}

// The same with x staged first.
template <int NPF, int KPF, int R, int NO>
__device__ __forceinline__ void resident_rowgemm_t(uint8_t* smem, const uint8_t* img, const float (&x)[R], float (&y)[NO]) {
  stage_rows(smem, x);
  resident_rowgemm_t_staged<NPF, KPF, R, NO>(smem, img, y);
}

// y = W x (before its bias) with the weights from a resident split image (W [NPF][KPF]) read K-major, x staged as a row
// tile and the result rows stored over it, one M half at a time.  smem is the warpgroup's kResidentStepBytes.
template <int NPF, int KPF, int R, int NO>
__device__ __forceinline__ void resident_rowgemm(uint8_t* smem, const uint8_t* img, const float (&x)[R], float (&y)[NO]) {
  constexpr int KP = pad16(R), NP = padn(NO);
  static_assert(KP == KPF && NP == NPF, "layer outside the resident image");
  static_assert(2 * 128 * KP * 2 <= kResidentStepBytes && NP * 128 * 4 <= kResidentStepBytes, "resident step plan");
  float* ys = reinterpret_cast<float*>(smem);
  stage_rows(smem, x);
  layer_mma<KP, NP, 0, true>(smem_u32(smem), 128 * KP * 2, image_operand<NPF, KPF, false>(img), ys, 4, kRowsGroupStride);
  sync();
  read_row<NO>(ys, 4, kRowsGroupStride, y);
}

// Two forward layers chained fragment to fragment: m = epi0(W0 x), y = W1 m (before its bias), both weights from the
// resident image (img0: W0 [NPF0][KPF0], img1: W1 [NPF1][NPF0]).  The first layer's MMAs end in registers (both M halves
// in flight); epi0(c, v) (column c of value v: the bias and ReLU) runs on them in fragment order, and they are stored as
// the second layer's A tile in place of the first's, split hi / lo.  Only the second layer's result goes back to rows.
// KEEP_MID (the backward, whose weight gradients and ReLU masks read m as rows): the first layer runs the row path
// instead, one M half at a time, with epi0 on the rows and m staged from them; its 64 live accumulators would add to the
// backward's spills (DESIGN.md section 4.3).  Both give the same bytes in the second layer's tile.  smem is the
// warpgroup's kResidentStepBytes.
template <int NPF0, int KPF0, int NPF1, bool KEEP_MID, int R, int NM, int NO, class Epi>
__device__ __forceinline__ void resident_chain(uint8_t* smem, const uint8_t* img0, const uint8_t* img1, const float (&x)[R],
                                               float (&mid)[NM], float (&y)[NO], Epi epi0) {
  constexpr int KP = pad16(R), NP = padn(NO);
  static_assert(KP == KPF0 && NM == NPF0 && NP == NPF1, "layers outside the resident image");
  static_assert(2 * 128 * NM * 2 <= kResidentStepBytes && 2 * 128 * KP * 2 <= kResidentStepBytes && NM * 128 * 4 <= kResidentStepBytes,
                "resident step plan");
  const uint32_t tile = smem_u32(smem);
  float* ys = reinterpret_cast<float*>(smem);
  if constexpr (KEEP_MID) {
    resident_rowgemm<NPF0, KPF0>(smem, img0, x, mid);
#pragma unroll
    for (int n = 0; n < NM; ++n) mid[n] = epi0(n, mid[n]);
    stage_rows(smem, mid);
  } else {
    stage_rows(smem, x);
    const int lane = tid() & 31;
    float d[2][NM / 2];
    layer_mma_frag<KP, NM, 0>(tile, 128 * KP * 2, image_operand<NPF0, KPF0, false>(img0), d);
    // fragment (i, j): column 8 i + 2 (lane % 4) + (j & 1)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < NM / 2; ++e) d[h][e] = epi0(8 * (e / 4) + 2 * (lane & 3) + (e & 1), d[h][e]);
    store_a_tile<NM>(tile, d);
    fence_proxy_async();
    sync();
  }
  layer_mma<NM, NP, 0, true>(tile, 128 * NM * 2, image_operand<NPF1, NM, false>(img1), ys, 4, kRowsGroupStride);
  sync();
  read_row<NO>(ys, 4, kRowsGroupStride, y);
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

// Weight gradient of the warpgroup's 128-point tile, gW[N][K] += dY^T X and gb[N] += column sums of dY, both operands
// read K-major over the points (the reduction dimension); accumulated in warpgroup registers and added to the global
// gradient once per tile.  Every thread of the CTA (one warpgroup) must call it.
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
  const int t = tid();
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

// ------------------------------------------------------------------------------------------
// On-chip weight gradients (ResidentLayers): dW / db of every tile are added to fp32 accumulators in shared memory,
// which the CTA adds to the global gradient once, at its end.
// ------------------------------------------------------------------------------------------

// Reduce-scatter over the warp of P values per lane (P a power of two <= 32): returns, in lane l, the sum over the 32
// lanes of v[l >> (5 - log2 P)].  P - 1 + (5 - log2 P) shuffles; v is clobbered.
template <int P, int S = 16>
__device__ __forceinline__ float warp_reduce_scatter(float* v, int lane) {
  if constexpr (S == 0) {
    return v[0];
  } else if constexpr (P == 1) {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], S);
    return warp_reduce_scatter<1, S / 2>(v, lane);
  } else {
    const bool up = (lane & S) != 0;
#pragma unroll
    for (int i = 0; i < P / 2; ++i) {
      const float send = up ? v[i] : v[i + P / 2], keep = up ? v[i + P / 2] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, S);
    }
    return warp_reduce_scatter<P / 2, S / 2>(v, lane);
  }
}

constexpr int pow2_at_least(int n) { return n <= 1 ? 1 : 2 * pow2_at_least((n + 1) / 2); }
constexpr int log2_exact(int n) { return n <= 1 ? 0 : 1 + log2_exact(n / 2); }

// put(i, sum over the warp's 32 lanes of v(i)) for i < M, in fp32 (32-value reduce-scatters; no serial loops), each i
// put by one lane.
template <int M, class V, class Put>
__device__ __forceinline__ void warp_column_sums(V v, Put put, int lane) {
#pragma unroll
  for (int c = 0; c < M; c += 32) {
    constexpr int kLeft = M % 32 == 0 ? 32 : M % 32;
    constexpr int P = pow2_at_least(M >= 32 ? 32 : kLeft);
    constexpr int SH = 5 - log2_exact(P);
    float u[P];
#pragma unroll
    for (int j = 0; j < P; ++j) u[j] = c + j < M ? v(c + j < M ? c + j : 0) : 0.f;
    const float s = warp_reduce_scatter<P>(u, lane);
    const int i = c + (lane >> SH);
    if ((lane & ((1 << SH) - 1)) == 0 && i < M) put(i, s);
  }
}

// A warpgroup's exclusive use of one accumulator: thread 0 takes the lock, the warpgroup's barrier passes it on.
__device__ __forceinline__ void acquire(int* lock) {
  if (tid() == 0) {
    while (atomicCAS(lock, 0, 1) != 0) __nanosleep(32);
    __threadfence_block();
  }
  sync();
}
__device__ __forceinline__ void release(int* lock) {
  __threadfence_block();
  sync();
  if (tid() == 0) {
    __threadfence_block();
    atomicExch(lock, 0);
  }
}

// Bytes of a warpgroup's dW operand region: the MN-major X tile of one weight_grad_acc round, hi | lo.  The fp32 heads'
// per-warp partial sums (kWarpPartial floats per warp) use the same region, which no MMA reads while a head runs.
// Floats of a layer's accumulator: dW in fragment order (the rows of warps that hold outputs n < N, KP / 2 floats per
// thread) followed by db[N].
constexpr int kDwXBytes = 16 * 1024;
constexpr int kWarpPartial = 256;
static_assert(4 * kWarpPartial * 4 <= kDwXBytes, "head partials within the dW operand region");
template <int K, int N>
struct DwAcc {
  static constexpr int KP = padn(K), kWarps = (N + 15) / 16;
  static constexpr int kW = kWarps * 32 * (KP / 2), kFloats = kW + N;
  // output n and input k of accumulator element e < kW
  static __device__ __forceinline__ void at(int e, int& n, int& k) {
    const int j = e & 3, f = e >> 2, lane = f & 31, wq = f >> 5, warp = wq / (KP / 8), q = wq % (KP / 8);
    n = 16 * warp + (lane >> 2) + (j >= 2 ? 8 : 0);
    k = 8 * q + 2 * (lane & 3) + (j & 1);
  }
};

// Weight gradient of the warpgroup's 128-point tile added to the layer's accumulator acc (DwAcc<K, N>), with dY staged
// once for it and for the layer's dx.  Every thread splits its dy row into the step tile `smem` as dx's K-major A tile
// (stage_rows' bytes: element (point p, output n) at (n / 8) * 2048 + p * 16 + (n % 8) * 2), which dW = dY^T X reads
// MN-major through the transpose bit; rows of dY past N read bytes that are never accumulated.  X goes MN-major into the
// dW operand region `xs` (16-byte split stores of 8 inputs of one point), PTS points per round: one round for KP <= 32,
// two 64-point rounds for KP = 64.  The k16 steps over all 128 points are one MMA chain, and the accumulator takes it
// under the layer's lock once per tile.  It is added before dx runs, so that its KP / 2 registers are not live next to
// dx's accumulators.  db: each warp's column sums of dy added to acc's bias row with shared-memory float adds, no lock.
// The dY tile is left in smem for resident_rowgemm_t_staged.  Every thread of the warpgroup must call it.
template <int K, int N>
__device__ __forceinline__ void weight_grad_acc(uint8_t* smem, uint8_t* xs, const float (&x)[K], const float (&dy)[N],
                                                float* acc, int* lock) {
  using A = DwAcc<K, N>;
  constexpr int KP = A::KP, YP = pad16(N);  // MMA width; dY tile width
  constexpr int PTS = kDwXBytes / (4 * KP) < 128 ? kDwXBytes / (4 * KP) : 128, ROUNDS = 128 / PTS;
  constexpr uint32_t YLO = 128 * YP * 2, XLO = PTS * KP * 2;
  static_assert(N <= 64 && 2 * YLO <= kResidentStepBytes && 2 * XLO <= kDwXBytes && PTS % 16 == 0, "dW plan");
  const int t = tid(), warp = t >> 5, lane = t & 31;
  float* db = acc + A::kW;
  warp_column_sums<N>([&](int n) { return dy[n]; }, [&](int n, float s) { atomicAdd(db + n, s); }, lane);
  sync();  // the previous readers of the step tile and of xs are done
#pragma unroll
  for (int c = 0; c < YP / 8; ++c) split_store_chunk(smem, smem + YLO, c * (128 * 16) + t * 16, dy, c);
  const uint32_t ay = smem_u32(smem), ax = smem_u32(xs);
  float d[KP / 2];
#pragma unroll
  for (int i = 0; i < KP / 2; ++i) d[i] = 0.f;
#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
    if (r > 0) {  // the previous round's MMAs are done with xs
      wait_all();
      sync();
    }
    if (t / PTS == r) {
#pragma unroll
      for (int c = 0; c < KP / 8; ++c) split_store_chunk(xs, xs + XLO, c * (PTS * 16) + (t % PTS) * 16, x, c);
    }
    fence_proxy_async();
    sync();
    fence_operands();
#pragma unroll
    for (int ks = 0; ks < PTS / 16; ++ks) {
      const uint32_t ya = ay + (r * (PTS / 16) + ks) * 256, xa = ax + ks * 256;
      const uint64_t dah = desc(ya, 128, 128 * 16), dal = desc(ya + YLO, 128, 128 * 16);
      const uint64_t dbh = desc(xa, 128, PTS * 16), dbl = desc(xa + XLO, 128, PTS * 16);
      mma_m64k16<KP, 1, 1>(d, dah, dbh, r > 0 || ks > 0);
      mma_m64k16<KP, 1, 1>(d, dal, dbh, 1);
      mma_m64k16<KP, 1, 1>(d, dah, dbl, 1);
      mma_m64k16<KP, 1, 1>(d, dal, dbl, 1);
    }
    commit();
  }
  wait_all();
  FNR_PHASE(kPhDw);
  acquire(lock);
  if (warp < A::kWarps) {
    float4* a4 = reinterpret_cast<float4*>(acc) + warp * (KP / 8) * 32 + lane;
#pragma unroll
    for (int q = 0; q < KP / 8; ++q) {
      float4 v = a4[q * 32];
      v.x += d[4 * q];
      v.y += d[4 * q + 1];
      v.z += d[4 * q + 2];
      v.w += d[4 * q + 3];
      a4[q * 32] = v;
    }
  }
  release(lock);
  FNR_PHASE(kPhDwFlush);
}

// Weight gradient of a narrow fp32 head (N = 1, 3 outputs) over the warpgroup's tile, exact fp32 on the CUDA cores: warp
// reduce-scatters of dy[n] x[k] and dy[n] into per-warp partials (part: 4 x kWarpPartial floats), then the warps' sums
// are added to acc ([N][K] then [N]).  Every thread of the warpgroup must call it.
template <int K, int N>
__device__ __forceinline__ void head_weight_grad_acc(float* part, const float (&x)[K], const float (&dy)[N], float* acc, int* lock) {
  static_assert(K % 32 == 0 && N * K + N <= kWarpPartial, "head partials");
  const int t = tid(), warp = t >> 5, lane = t & 31;
  float* pw = part + warp * kWarpPartial;
#pragma unroll
  for (int n = 0; n < N; ++n) warp_column_sums<K>([&](int k) { return dy[n] * x[k]; }, [&](int k, float s) { pw[n * K + k] = s; }, lane);
  warp_column_sums<N>([&](int n) { return dy[n]; }, [&](int n, float s) { pw[N * K + n] = s; }, lane);
  acquire(lock);  // its barrier also orders the partial stores before the reads below
  for (int e = t; e < N * K + N; e += 128)
    acc[e] += part[e] + part[kWarpPartial + e] + part[2 * kWarpPartial + e] + part[3 * kWarpPartial + e];
  release(lock);
}

}  // namespace wg
}  // namespace fnr
