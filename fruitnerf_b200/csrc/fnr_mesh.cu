// Surface meshes of a trained scene (`ns-export-semantics tsdf`, nerfstudio ns-export tsdf):
//   tsdf_integrate_kernel  one thread per grid point fuses a batch of rendered frames in frame order: project, look up the
//                          pixel's ray distance, convert it to depth along the optical axis, update the truncated signed
//                          distance, colour and fruit probability with count weights.  No atomics: the result is the
//                          sequential per-image update whatever the launch order.
//   mc_count_kernel        marching cubes, pass 1: per 2^16-point chunk, each point's active edges (a vertex each) and
//                          the triangle count of the cell it is the min corner of; the chunk-local vertex offset of every
//                          point (with its 3-bit edge mask) and the chunk totals go to scratch
//   mc_scan_kernel         exclusive scan of the chunk totals (one block), and the mesh's vertex and face counts
//   mc_emit_kernel         pass 2: vertices (position, gradient normal, nearest-point colour and fruit) and faces in
//                          (point, axis) and (cell, table) order, at offsets from a block scan of each round
// Every operation whose rounding matters is written out (__fmul_rn, __fadd_rn, __fdiv_rn, __fsqrt_rn) so that
// mesh.restated_integrate / mesh.marching_cubes_numpy are the exact reference.  Counts and indices are int64.
#include "fnr_common.cuh"
#include "fnr_kernels.h"
#include "fnr_mesh_table.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kMcThreads = 1024;
constexpr int kChunkShift = 16;  // points per marching-cubes chunk: 2^16 = 64 rounds of kMcThreads
constexpr int kRounds = (1 << kChunkShift) / kMcThreads;
constexpr uint32_t kLocalMask = (1u << 29) - 1;  // vloc word: chunk-local vertex offset | edge mask << 29

struct KTsdf {
  float *values, *weights, *colors, *fruit;  // [N], [N], [N,3], [N] or NULL
  long long nx, ny, nz;
  float origin[3], voxel[3], trunc;
  const float* c2w;  // [B,3,4]
  const float *fx, *fy, *cx, *cy;  // [B]
  const float* depth;  // [B,H,W] ray distance
  const float* rgb;    // [B,H,W,3]
  const float* frame_fruit;  // [B,H,W] or NULL
  int B, H, W;
};

__global__ void __launch_bounds__(kThreads) tsdf_integrate_kernel(KTsdf A) {
  const long long N = A.nx * A.ny * A.nz;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (long long)gridDim.x * blockDim.x) {
    const long long k = p % A.nz, q = p / A.nz, j = q % A.ny, i = q / A.ny;
    const float x[3] = {__fadd_rn(A.origin[0], __fmul_rn((float)i, A.voxel[0])), __fadd_rn(A.origin[1], __fmul_rn((float)j, A.voxel[1])),
                        __fadd_rn(A.origin[2], __fmul_rn((float)k, A.voxel[2]))};
    float val = A.values[p], w = A.weights[p];
    float c0 = A.colors[3 * p], c1 = A.colors[3 * p + 1], c2 = A.colors[3 * p + 2];
    float fr = A.frame_fruit ? A.fruit[p] : 0.f;
    bool touched = false;
    for (int b = 0; b < A.B; ++b) {
      const float* m = A.c2w + 12 * (size_t)b;  // [3][4] row-major: R | t
      const float d0 = __fsub_rn(x[0], __ldg(m + 3)), d1 = __fsub_rn(x[1], __ldg(m + 7)), d2 = __fsub_rn(x[2], __ldg(m + 11));
      float pc[3];
#pragma unroll
      for (int c = 0; c < 3; ++c)  // R^T (x - t)
        pc[c] = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + c), d0), __fmul_rn(__ldg(m + 4 + c), d1)), __fmul_rn(__ldg(m + 8 + c), d2));
      const float zc = -pc[2];
      if (!(zc > 0.f)) continue;
      const float fx = __ldg(A.fx + b), fy = __ldg(A.fy + b), cx = __ldg(A.cx + b), cy = __ldg(A.cy + b);
      const float u = __fadd_rn(cx, __fdiv_rn(__fmul_rn(fx, pc[0]), zc));
      const float v = __fsub_rn(cy, __fdiv_rn(__fmul_rn(fy, pc[1]), zc));
      if (!(u >= 0.f && u < (float)A.W && v >= 0.f && v < (float)A.H)) continue;
      const int col = (int)floorf(u), row = (int)floorf(v);
      const size_t pix = ((size_t)b * A.H + row) * A.W + col;
      const float t = __ldg(A.depth + pix);
      if (!(t > 0.f)) continue;
      // ray distance -> depth along the optical axis, with the pixel-centre direction
      const float a = __fdiv_rn(__fsub_rn(__fadd_rn((float)col, 0.5f), cx), fx);
      const float e = __fdiv_rn(__fsub_rn(__fadd_rn((float)row, 0.5f), cy), fy);
      const float zpix = __fdiv_rn(t, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(e, e)), 1.f)));
      const float sdf = __fsub_rn(zpix, zc);
      if (!(sdf > -A.trunc)) continue;
      const float tsdf = fminf(fmaxf(__fdiv_rn(sdf, A.trunc), -1.f), 1.f);
      const float w1 = __fadd_rn(w, 1.f);
      val = __fdiv_rn(__fadd_rn(__fmul_rn(val, w), tsdf), w1);
      c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, w), __ldg(A.rgb + 3 * pix)), w1);
      c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, w), __ldg(A.rgb + 3 * pix + 1)), w1);
      c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, w), __ldg(A.rgb + 3 * pix + 2)), w1);
      if (A.frame_fruit) fr = __fdiv_rn(__fadd_rn(__fmul_rn(fr, w), __ldg(A.frame_fruit + pix)), w1);
      w = w1;
      touched = true;
    }
    if (touched) {
      A.values[p] = val;
      A.weights[p] = w;
      A.colors[3 * p] = c0;
      A.colors[3 * p + 1] = c1;
      A.colors[3 * p + 2] = c2;
      if (A.frame_fruit) A.fruit[p] = fr;
    }
  }
}

struct KMc {
  const float* values;  // [X,Y,Z]
  long long dim[3];
  long long stride[3];  // Y*Z, Z, 1
  long long N;
  unsigned long long* chunk_v;  // [C] vertices per chunk, then their exclusive scan
  unsigned long long* chunk_f;  // [C] faces per chunk, then their exclusive scan
  uint32_t* vloc;               // [N]
  int64_t* totals;              // [2] vertices, faces
  long long num_chunks;
  // emit
  const float *colors, *fruit;  // [N,3], [N] or NULL
  float origin[3], voxel[3];
  float *vertices, *normals, *vertex_colors, *vertex_fruit;
  int64_t* faces;  // [F,3]
};

__device__ __forceinline__ bool inside(const float* v, long long p) { return __ldg(v + p) < 0.f; }

// Exclusive block scan (blockDim.x == kMcThreads) of x; `total` gets the block's sum.  s_warp: 32 entries of shared memory.
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T x, T* s_warp, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    T w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  const T before = warp ? s_warp[warp - 1] : T(0);
  total = s_warp[31];
  __syncthreads();  // s_warp is reused by the next call
  return before + inc - x;
}

// Point p = (i,j,k): its 3-bit mask of active edges (bit a: the edge p -> p + e_a has one inside endpoint) and, when p is
// the min corner of a cell, the cell's case (else -1).
__device__ __forceinline__ void point_edges_and_case(const KMc& A, long long p, int& mask, int& cs) {
  const long long k = p % A.dim[2], q = p / A.dim[2], j = q % A.dim[1], i = q / A.dim[1];
  const bool has[3] = {i < A.dim[0] - 1, j < A.dim[1] - 1, k < A.dim[2] - 1};
  const bool in0 = inside(A.values, p);
  mask = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (has[a] && inside(A.values, p + A.stride[a]) != in0) mask |= 1 << a;
  cs = -1;
  if (has[0] && has[1] && has[2]) {
    cs = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const long long pc = p + (c & 1) * A.stride[0] + ((c >> 1) & 1) * A.stride[1] + ((c >> 2) & 1) * A.stride[2];
      cs |= (int)inside(A.values, pc) << c;
    }
  }
}

__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(KMc A) {
  __shared__ int8_t s_count[256];
  __shared__ uint32_t s_warp[32];
  if (threadIdx.x < 256) s_count[threadIdx.x] = kMcTriCount[threadIdx.x];
  __syncthreads();
  const long long base = (long long)blockIdx.x << kChunkShift;
  uint32_t run_v = 0, run_f = 0;
  for (int r = 0; r < kRounds; ++r) {
    const long long p = base + r * kMcThreads + threadIdx.x;
    int mask = 0, cs = -1;
    if (p < A.N) point_edges_and_case(A, p, mask, cs);
    const uint32_t nv = __popc(mask), nf = cs >= 0 ? (uint32_t)s_count[cs] : 0u;
    uint32_t total;
    const uint32_t excl = block_exclusive_scan<uint32_t>(nv | nf << 16, s_warp, total);  // both halves stay below 2^16
    if (p < A.N) A.vloc[p] = (run_v + (excl & 0xffffu)) | (uint32_t)mask << 29;
    run_v += total & 0xffffu;
    run_f += total >> 16;
  }
  if (threadIdx.x == 0) {
    A.chunk_v[blockIdx.x] = run_v;
    A.chunk_f[blockIdx.x] = run_f;
  }
}

__global__ void __launch_bounds__(kMcThreads) mc_scan_kernel(KMc A) {
  __shared__ unsigned long long s_warp[32];
  unsigned long long run_v = 0, run_f = 0;
  for (long long t0 = 0; t0 < A.num_chunks; t0 += kMcThreads) {
    const long long t = t0 + threadIdx.x;
    const unsigned long long v = t < A.num_chunks ? A.chunk_v[t] : 0ull, f = t < A.num_chunks ? A.chunk_f[t] : 0ull;
    unsigned long long tv, tf;
    const unsigned long long ev = block_exclusive_scan<unsigned long long>(v, s_warp, tv);
    const unsigned long long ef = block_exclusive_scan<unsigned long long>(f, s_warp, tf);
    if (t < A.num_chunks) {
      A.chunk_v[t] = run_v + ev;
      A.chunk_f[t] = run_f + ef;
    }
    run_v += tv;
    run_f += tf;
  }
  if (threadIdx.x == 0) {
    A.totals[0] = (long long)run_v;
    A.totals[1] = (long long)run_f;
  }
}

// id of the vertex on the edge q -> q + e_a (which must be active)
__device__ __forceinline__ long long vertex_id(const KMc& A, long long q, int a) {
  const uint32_t word = A.vloc[q];
  return (long long)A.chunk_v[q >> kChunkShift] + (word & kLocalMask) + __popc((word >> 29) & ((1u << a) - 1u));
}

// d values / d axis b at grid point q (index ib on that axis), in world units
__device__ __forceinline__ float grad_axis(const KMc& A, long long q, long long ib, int b) {
  const float* v = A.values;
  const long long s = A.stride[b];
  float g;
  if (ib == 0) g = __fsub_rn(__ldg(v + q + s), __ldg(v + q));
  else if (ib == A.dim[b] - 1) g = __fsub_rn(__ldg(v + q), __ldg(v + q - s));
  else g = __fmul_rn(__fsub_rn(__ldg(v + q + s), __ldg(v + q - s)), 0.5f);
  return __fdiv_rn(g, A.voxel[b]);
}

__device__ void emit_vertex(const KMc& A, long long p, const long long idx[3], int a, long long id) {
  const long long pb = p + A.stride[a];
  const float va = __ldg(A.values + p), vb = __ldg(A.values + pb);
  const float s = __fdiv_rn(__fsub_rn(0.f, va), __fsub_rn(vb, va));
  float coord[3], n[3];
  long long near = 0;
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    coord[b] = (float)idx[b];
    if (b == a) coord[b] = __fadd_rn(coord[b], s);
    A.vertices[3 * id + b] = __fadd_rn(A.origin[b], __fmul_rn(coord[b], A.voxel[b]));
    long long r = (long long)rintf(coord[b]);  // numpy round: half to even
    r = r < 0 ? 0 : (r > A.dim[b] - 1 ? A.dim[b] - 1 : r);
    near += r * A.stride[b];
    const long long ib = idx[b] + (b == a);
    const float ga = grad_axis(A, p, idx[b], b), gb = grad_axis(A, pb, ib, b);
    n[b] = __fadd_rn(ga, __fmul_rn(s, __fsub_rn(gb, ga)));
  }
  const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
  // a vanishing gradient (a one-voxel sliver between clamped plateaus) falls back to the edge, toward its outside end
#pragma unroll
  for (int b = 0; b < 3; ++b) A.normals[3 * id + b] = len > 0.f ? __fdiv_rn(n[b], len) : (b == a ? (vb > va ? 1.f : -1.f) : 0.f);
  if (A.vertex_colors) {
#pragma unroll
    for (int b = 0; b < 3; ++b) A.vertex_colors[3 * id + b] = __ldg(A.colors + 3 * near + b);
  }
  if (A.vertex_fruit) A.vertex_fruit[id] = __ldg(A.fruit + near);
}

__global__ void __launch_bounds__(kMcThreads) mc_emit_kernel(KMc A) {
  __shared__ int8_t s_count[256];
  __shared__ int8_t s_table[256][3 * kMcMaxTriangles];
  __shared__ int8_t s_edge[12][4];
  __shared__ uint32_t s_warp[32];
  for (int t = threadIdx.x; t < 256 * 3 * kMcMaxTriangles; t += blockDim.x) (&s_table[0][0])[t] = (&kMcTriTable[0][0])[t];
  if (threadIdx.x < 256) s_count[threadIdx.x] = kMcTriCount[threadIdx.x];
  if (threadIdx.x < 48) (&s_edge[0][0])[threadIdx.x] = (&kMcEdge[0][0])[threadIdx.x];
  __syncthreads();
  const long long base = (long long)blockIdx.x << kChunkShift;
  const long long fbase = (long long)A.chunk_f[blockIdx.x];
  uint32_t run_f = 0;
  for (int r = 0; r < kRounds; ++r) {
    const long long p = base + r * kMcThreads + threadIdx.x;
    int cs = -1;
    if (p < A.N) {
      const uint32_t word = A.vloc[p];
      const int mask = (int)(word >> 29);
      const long long k = p % A.dim[2], q = p / A.dim[2], j = q % A.dim[1], i = q / A.dim[1];
      const long long idx[3] = {i, j, k};
      if (mask) {
        long long id = (long long)A.chunk_v[blockIdx.x] + (word & kLocalMask);
        for (int a = 0; a < 3; ++a)
          if (mask >> a & 1) emit_vertex(A, p, idx, a, id++);
      }
      if (i < A.dim[0] - 1 && j < A.dim[1] - 1 && k < A.dim[2] - 1) {
        cs = 0;
#pragma unroll
        for (int c = 0; c < 8; ++c)
          cs |= (int)inside(A.values, p + (c & 1) * A.stride[0] + ((c >> 1) & 1) * A.stride[1] + ((c >> 2) & 1) * A.stride[2]) << c;
      }
    }
    const uint32_t nf = cs >= 0 ? (uint32_t)s_count[cs] : 0u;
    uint32_t total;
    const uint32_t excl = block_exclusive_scan<uint32_t>(nf, s_warp, total);
    if (nf) {
      int64_t* out = A.faces + 3 * (fbase + run_f + excl);
      for (int t = 0; t < (int)nf * 3; ++t) {
        const int8_t* e = s_edge[s_table[cs][t]];
        out[t] = vertex_id(A, p + e[0] * A.stride[0] + e[1] * A.stride[1] + e[2] * A.stride[2], e[3]);
      }
    }
    run_f += total;
  }
}

bool finite_positive3(const float* v) {
  return v && isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]) && v[0] > 0.f && v[1] > 0.f && v[2] > 0.f;
}

bool finite3(const float* v) { return v && isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]); }

// dims >= 2 on every axis and few enough points for 2^31 - 1 chunks of 2^16
bool valid_dims(int64_t nx, int64_t ny, int64_t nz) {
  if (nx < 2 || ny < 2 || nz < 2) return false;
  const long double n = (long double)nx * ny * nz;
  return n < (long double)(1LL << 46);
}

KMc mc_args(const float* values, int64_t nx, int64_t ny, int64_t nz, const void* scratch) {
  KMc A{};
  A.values = values;
  A.dim[0] = nx, A.dim[1] = ny, A.dim[2] = nz;
  A.stride[0] = ny * nz, A.stride[1] = nz, A.stride[2] = 1;
  A.N = nx * ny * nz;
  A.num_chunks = (A.N + (1LL << kChunkShift) - 1) >> kChunkShift;
  char* s = (char*)scratch;
  A.chunk_v = (unsigned long long*)s;
  A.chunk_f = A.chunk_v + A.num_chunks;
  A.vloc = (uint32_t*)(A.chunk_f + A.num_chunks);
  return A;
}

size_t mc_scratch_bytes(int64_t nx, int64_t ny, int64_t nz) {
  const long long N = nx * ny * nz, C = (N + (1LL << kChunkShift) - 1) >> kChunkShift;
  return (size_t)C * 16 + (size_t)N * 4;
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_tsdf_integrate(float* values, float* weights, float* colors, float* fruit, int64_t nx, int64_t ny, int64_t nz, const float* origin,
                       const float* voxel_size, float truncation, const float* c2w, const float* fx, const float* fy, const float* cx,
                       const float* cy, const float* depth, const float* rgb, const float* frame_fruit, int32_t num_frames, int32_t height,
                       int32_t width, void* stream) {
  if (!values || !weights || !colors || (frame_fruit && !fruit) || !c2w || !fx || !fy || !cx || !cy || !depth || !rgb ||
      !valid_dims(nx, ny, nz) || !finite3(origin) || !finite_positive3(voxel_size) || !isfinite(truncation) || !(truncation > 0.f) ||
      height <= 0 || width <= 0 || num_frames < 0) {
    set_error("invalid arguments to fnr_tsdf_integrate (grid %lldx%lldx%lld, %d frames of %dx%d, truncation %g)", (long long)nx, (long long)ny,
              (long long)nz, num_frames, width, height, (double)truncation);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_frames == 0) return FNR_OK;
  KTsdf A{values, weights, colors, fruit, nx, ny, nz, {origin[0], origin[1], origin[2]}, {voxel_size[0], voxel_size[1], voxel_size[2]},
          truncation, c2w, fx, fy, cx, cy, depth, rgb, frame_fruit, num_frames, height, width};
  const long long N = (long long)nx * ny * nz;
  tsdf_integrate_kernel<<<grid_for(N, kThreads, sm_count() * 32), kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A);
  return check_launch("tsdf_integrate_kernel");
}

int fnr_marching_cubes_scratch_bytes(int64_t nx, int64_t ny, int64_t nz, size_t* bytes) {
  if (!bytes || !valid_dims(nx, ny, nz)) {
    set_error("invalid arguments to fnr_marching_cubes_scratch_bytes (grid %lldx%lldx%lld)", (long long)nx, (long long)ny, (long long)nz);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  *bytes = mc_scratch_bytes(nx, ny, nz);
  return FNR_OK;
}

int fnr_marching_cubes_count(const float* values, int64_t nx, int64_t ny, int64_t nz, void* scratch, size_t scratch_bytes, int64_t* totals,
                             void* stream) {
  if (!values || !scratch || !totals || !valid_dims(nx, ny, nz) || scratch_bytes < mc_scratch_bytes(nx, ny, nz)) {
    set_error("invalid arguments to fnr_marching_cubes_count (grid %lldx%lldx%lld, %zu scratch bytes)", (long long)nx, (long long)ny, (long long)nz,
              scratch_bytes);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KMc A = mc_args(values, nx, ny, nz, scratch);
  A.totals = totals;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  mc_count_kernel<<<(unsigned)A.num_chunks, kMcThreads, 0, st>>>(A);
  if (int rc = check_launch("mc_count_kernel")) return rc;
  mc_scan_kernel<<<1, kMcThreads, 0, st>>>(A);
  return check_launch("mc_scan_kernel");
}

int fnr_marching_cubes_emit(const float* values, const float* colors, const float* fruit, int64_t nx, int64_t ny, int64_t nz, const float* origin,
                            const float* voxel_size, const void* scratch, size_t scratch_bytes, int64_t num_vertices, int64_t num_faces,
                            float* vertices, float* normals, float* vertex_colors, float* vertex_fruit, int64_t* faces, void* stream) {
  if (!values || !scratch || !valid_dims(nx, ny, nz) || scratch_bytes < mc_scratch_bytes(nx, ny, nz) || !finite3(origin) ||
      !finite_positive3(voxel_size) || num_vertices < 0 || num_faces < 0) {
    set_error("invalid arguments to fnr_marching_cubes_emit (grid %lldx%lldx%lld, %lld vertices, %lld faces)", (long long)nx, (long long)ny,
              (long long)nz, (long long)num_vertices, (long long)num_faces);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_vertices > 0x7fffffffLL) {
    set_error("fnr_marching_cubes_emit: %lld vertices exceed the 2^31 - 1 a PLY int face index can address", (long long)num_vertices);
    return FNR_ERR_UNSUPPORTED;
  }
  if ((num_vertices > 0 && (!vertices || !normals || !colors != !vertex_colors || !fruit != !vertex_fruit)) || (num_faces > 0 && !faces)) {
    set_error("fnr_marching_cubes_emit: NULL outputs for %lld vertices and %lld faces", (long long)num_vertices, (long long)num_faces);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_vertices == 0) return FNR_OK;  // no active edge: no vertex, no face
  KMc A = mc_args(values, nx, ny, nz, const_cast<void*>(scratch));
  A.colors = colors;
  A.fruit = fruit;
  for (int b = 0; b < 3; ++b) {
    A.origin[b] = origin[b];
    A.voxel[b] = voxel_size[b];
  }
  A.vertices = vertices;
  A.normals = normals;
  A.vertex_colors = colors ? vertex_colors : nullptr;
  A.vertex_fruit = fruit ? vertex_fruit : nullptr;
  A.faces = faces;
  mc_emit_kernel<<<(unsigned)A.num_chunks, kMcThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(A);
  return check_launch("mc_emit_kernel");
}

}  // extern "C"
