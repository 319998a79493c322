// The `charts` UV unwrap of NeRF-textured meshes (`--unwrap-method charts`; DESIGN section 4.3r).  Faces are grouped into
// connected charts of one dominant signed normal axis, each chart is projected onto its axis plane at one shared scale of
// texels per unit length, and the charts are packed into one square atlas:
//   prepare_kernel         per face: refuses face indices outside [0, V) and non-finite vertices (one device flag), the
//                          label (dominant signed axis of the right-hand normal), the projected corners and the 3F
//                          half-edge keys (fnr_mesh_edges.cuh), sorted once
//   link_kernel            per interior edge (a run of exactly two half-edges): unites its faces (fnr_union_find.cuh) when
//                          their labels agree and neither face has been cut into a chart of its own
//   flatten / root / chart chart id = rank of the chart's smallest face index (an exclusive scan of the root flags)
//   extent_kernel          per face: atomic min / max of the projected corners per chart (order-free, so exact)
//   (host)                 next-fit shelf packing of the charts' rectangles, the scale by fp64 bisection
//   uv_kernel              per face: texel coordinates of its corners and its texel box grown by the gutter
//   conflict / mark        per (face, texel of its box): texel centres strictly inside two triangles; every face there but
//                          the smallest becomes a chart of its own, and the charts are built again
//   owner_kernel           per (face, texel of its box): 64-bit atomicMin of (fp32 squared distance bits, face) within the
//                          gutter
//   compact_kernel         owned texels in texel order (an exclusive scan): owner map, face and barycentrics per texel
// Every fp64 operation is rounded where written (no FMA), so texture.py restates the unwrap bit for bit.  The host reads
// a few integers and the charts' extents per round and allocates nothing on the device: one caller-sized scratch.
#include <cub/cub.cuh>
#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <numeric>
#include <vector>
#include "fnr_common.cuh"
#include "fnr_kernels.h"
#include "fnr_mesh_edges.cuh"
#include "fnr_union_find.cuh"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr long long kMaxIndex = 2147483647LL;
constexpr long long kMaxFaces = kMaxIndex / 3;  // 3F half-edges are sorted as one int-sized cub call
constexpr int kMargin = FNR_UNWRAP_MARGIN;
constexpr double kGutter = FNR_UNWRAP_GUTTER;
constexpr unsigned long long kNoOwner = ~0ull;

// projected axes (texel x, texel y) per label +x, -x, +y, -y, +z, -z: every face keeps a positive area in vt space
__constant__ int c_axes[6][2] = {{2, 1}, {1, 2}, {0, 2}, {2, 0}, {1, 0}, {0, 1}};

// doubles as unsigned keys whose integer order is their numeric order (+0 and -0 never occur: positions are x + 0)
__device__ __forceinline__ unsigned long long okey(double x) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(x);
  return (b >> 63) ? ~b : b | 0x8000000000000000ull;
}
__device__ __forceinline__ double okey_inv(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? k & 0x7FFFFFFFFFFFFFFFull : ~k));
}

struct KPrepare {
  const float* vertices;  // [V,3]
  const int64_t* faces;   // [F,3]
  long long V, F;
  int32_t* labels;          // [F]
  double* proj;             // [F,3,2]
  unsigned long long* keys;  // [3F]
  int* vals;                 // [3F]
  int* bad;
};

__global__ void __launch_bounds__(kThreads) prepare_kernel(KPrepare A) {
  for (long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x; f < A.F; f += (long long)gridDim.x * blockDim.x) {
    long long idx[3];
    double P[3][3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      idx[c] = A.faces[3 * f + c];
      ok = ok && idx[c] >= 0 && idx[c] < A.V;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float x = ok ? A.vertices[3 * idx[c] + k] : 0.f;
        ok = ok && isfinite(x);
        P[c][k] = __dadd_rn((double)x, 0.0);
      }
    if (!ok) {
      atomicExch(A.bad, 1);
      continue;
    }
    double e1[3], e2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      e1[k] = __dsub_rn(P[1][k], P[0][k]);
      e2[k] = __dsub_rn(P[2][k], P[0][k]);
    }
    const double n0 = __dsub_rn(__dmul_rn(e1[1], e2[2]), __dmul_rn(e1[2], e2[1]));
    const double n1 = __dsub_rn(__dmul_rn(e1[2], e2[0]), __dmul_rn(e1[0], e2[2]));
    const double n2 = __dsub_rn(__dmul_rn(e1[0], e2[1]), __dmul_rn(e1[1], e2[0]));
    int k = 0;
    double best = fabs(n0), nk = n0;
    if (fabs(n1) > best) {
      k = 1;
      best = fabs(n1);
      nk = n1;
    }
    if (fabs(n2) > best) {
      k = 2;
      nk = n2;
    }
    const int label = 2 * k + (nk < 0.0);
    A.labels[f] = label;
    const int ca = c_axes[label][0], cb = c_axes[label][1];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      A.proj[6 * f + 2 * c] = ca == 0 ? P[c][0] : ca == 1 ? P[c][1] : P[c][2];
      A.proj[6 * f + 2 * c + 1] = cb == 0 ? P[c][0] : cb == 1 ? P[c][1] : P[c][2];
      A.keys[3 * f + c] = half_edge_key(idx[c], idx[c == 2 ? 0 : c + 1], A.V);
      A.vals[3 * f + c] = (int)(3 * f + c);
    }
  }
}

__global__ void __launch_bounds__(kThreads) iota_kernel(int* a, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) a[i] = (int)i;
}

// an interior edge is a run of exactly two equal keys; it joins its faces when their labels agree and neither is cut
__global__ void __launch_bounds__(kThreads) link_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ vals, long long E,
                                                        const int32_t* __restrict__ labels, const int* __restrict__ cut, int* parent) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if ((i > 0 && keys[i - 1] == k) || i + 1 >= E || keys[i + 1] != k || (i + 2 < E && keys[i + 2] == k)) continue;
    const int a = vals[i] / 3, b = vals[i + 1] / 3;
    if (labels[a] == labels[b] && !cut[a] && !cut[b]) unite(parent, a, b);
  }
}

// every node straight at its root (as fnr_cluster.cu's flatten: no hooking is in flight, each thread writes its own slot),
// and the root flags
__global__ void __launch_bounds__(kThreads) flatten_kernel(int* parent, int* flag, long long F) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < F; i += (long long)gridDim.x * blockDim.x) {
    const volatile int* p = parent;
    int r = p[i];
    while (r != p[r]) r = p[r];
    parent[i] = r;
    flag[i] = r == (int)i;
  }
}

__global__ void __launch_bounds__(kThreads) chart_kernel(const int* __restrict__ parent, const int* __restrict__ rank, long long F,
                                                         int32_t* __restrict__ chart, unsigned long long* __restrict__ lo,
                                                         unsigned long long* __restrict__ hi) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < F; i += (long long)gridDim.x * blockDim.x) {
    chart[i] = rank[parent[i]];
    lo[2 * i] = lo[2 * i + 1] = ~0ull;  // chart slots: at most F charts
    hi[2 * i] = hi[2 * i + 1] = 0ull;
  }
}

__global__ void __launch_bounds__(kThreads) extent_kernel(const double* __restrict__ proj, const int32_t* __restrict__ chart, long long F,
                                                          unsigned long long* lo, unsigned long long* hi) {
  for (long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    const int c = chart[f];
#pragma unroll
    for (int ax = 0; ax < 2; ++ax) {
      const double p0 = proj[6 * f + ax], p1 = proj[6 * f + 2 + ax], p2 = proj[6 * f + 4 + ax];
      atomicMin(lo + 2 * c + ax, okey(fmin(fmin(p0, p1), p2)));
      atomicMax(hi + 2 * c + ax, okey(fmax(fmax(p0, p1), p2)));
    }
  }
}

// ext[c] = (max - min) per axis, pmin[c] = min per axis
__global__ void __launch_bounds__(kThreads) extent_finish_kernel(const unsigned long long* __restrict__ lo, const unsigned long long* __restrict__ hi,
                                                                 long long C, double* __restrict__ ext, double* __restrict__ pmin) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < 2 * C; i += (long long)gridDim.x * blockDim.x) {
    const double a = okey_inv(lo[i]), b = okey_inv(hi[i]);
    pmin[i] = a;
    ext[i] = __dsub_rn(b, a);
  }
}

// texel coordinates offset + m + s (p - p_min) of every corner, and the face's texel box grown by the gutter:
// columns j with j + 0.5 in [x_min - g, x_max + g], likewise rows, clamped to the atlas
__global__ void __launch_bounds__(kThreads) uv_kernel(const double* __restrict__ proj, const int32_t* __restrict__ chart,
                                                      const int32_t* __restrict__ offsets, const double* __restrict__ pmin, double s,
                                                      long long F, int N, double* __restrict__ uv, int* __restrict__ box,
                                                      long long* __restrict__ boxn) {
  for (long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    const int c = chart[f];
    int lo[2], len[2];
#pragma unroll
    for (int ax = 0; ax < 2; ++ax) {
      const double o = (double)(offsets[2 * c + ax] + kMargin), m = pmin[2 * c + ax];
      double mn = 0.0, mx = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double x = __dadd_rn(o, __dmul_rn(s, __dsub_rn(proj[6 * f + 2 * k + ax], m)));
        uv[6 * f + 2 * k + ax] = x;
        mn = k == 0 ? x : fmin(mn, x);
        mx = k == 0 ? x : fmax(mx, x);
      }
      const int a = max((int)ceil(__dsub_rn(mn, kGutter + 0.5)), 0), b = min((int)floor(__dadd_rn(mx, kGutter - 0.5)), N - 1);
      lo[ax] = a;
      len[ax] = max(b - a + 1, 0);
    }
    box[4 * f] = lo[0];
    box[4 * f + 1] = lo[1];
    box[4 * f + 2] = len[0];
    box[4 * f + 3] = len[1];
    boxn[f] = (long long)len[0] * len[1];
  }
}

// (c - a) x (b - a) in texel space: > 0 on the inner side of edge a -> b of a face (faces have negative area in texel
// space, positive in vt space)
__device__ __forceinline__ double edge_fn(double ax, double ay, double bx, double by, double cx, double cy) {
  return __dsub_rn(__dmul_rn(__dsub_rn(cx, ax), __dsub_rn(by, ay)), __dmul_rn(__dsub_rn(cy, ay), __dsub_rn(bx, ax)));
}

struct Tri {
  double x[3], y[3];
};

__device__ __forceinline__ void load_tri(const double* uv, long long f, Tri& t) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    t.x[k] = uv[6 * f + 2 * k];
    t.y[k] = uv[6 * f + 2 * k + 1];
  }
}

__device__ __forceinline__ bool strictly_inside(const Tri& t, double cx, double cy) {
  return edge_fn(t.x[1], t.y[1], t.x[2], t.y[2], cx, cy) > 0.0 && edge_fn(t.x[2], t.y[2], t.x[0], t.y[0], cx, cy) > 0.0 &&
         edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], cx, cy) > 0.0;
}

// squared distance from c to the triangle and the fp32 barycentrics of its closest point (the header's order)
__device__ __forceinline__ double closest(const Tri& t, double cx, double cy, float& w0, float& w1, float& w2) {
  const double e0 = edge_fn(t.x[1], t.y[1], t.x[2], t.y[2], cx, cy);
  const double e1 = edge_fn(t.x[2], t.y[2], t.x[0], t.y[0], cx, cy);
  const double e2 = edge_fn(t.x[0], t.y[0], t.x[1], t.y[1], cx, cy);
  const double sum = __dadd_rn(__dadd_rn(e0, e1), e2);
  if (e0 >= 0.0 && e1 >= 0.0 && e2 >= 0.0 && sum > 0.0) {
    w1 = __double2float_rn(__ddiv_rn(e1, sum));
    w2 = __double2float_rn(__ddiv_rn(e2, sum));
    w0 = fmaxf(__fsub_rn(__fsub_rn(1.f, w1), w2), 0.f);
    return 0.0;
  }
  double best = 0.0, bt = 0.0;
  int bk = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int k1 = k == 2 ? 0 : k + 1;
    const double dx = __dsub_rn(t.x[k1], t.x[k]), dy = __dsub_rn(t.y[k1], t.y[k]);
    const double l2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
    const double num = __dadd_rn(__dmul_rn(__dsub_rn(cx, t.x[k]), dx), __dmul_rn(__dsub_rn(cy, t.y[k]), dy));
    const double tt = l2 > 0.0 ? fmin(fmax(__ddiv_rn(num, l2 > 0.0 ? l2 : 1.0), 0.0), 1.0) : 0.0;
    const double qx = __dsub_rn(cx, __dadd_rn(t.x[k], __dmul_rn(tt, dx))), qy = __dsub_rn(cy, __dadd_rn(t.y[k], __dmul_rn(tt, dy)));
    const double d2 = __dadd_rn(__dmul_rn(qx, qx), __dmul_rn(qy, qy));
    if (k == 0 || d2 < best) {
      best = d2;
      bt = tt;
      bk = k;
    }
  }
  if (sum > 0.0) {
    const float wt = __double2float_rn(bt);
    w0 = bk == 0 ? __fsub_rn(1.f, wt) : bk == 2 ? wt : 0.f;
    w1 = bk == 1 ? __fsub_rn(1.f, wt) : bk == 0 ? wt : 0.f;
    w2 = bk == 2 ? __fsub_rn(1.f, wt) : bk == 1 ? wt : 0.f;
  } else {  // a degenerate triangle: vertex 0
    w0 = 1.f;
    w1 = 0.f;
    w2 = 0.f;
  }
  return best;
}

// the face and texel of work item r: the last face whose box starts at or before r (binary search of the exclusive scan)
__device__ __forceinline__ long long work_face(const long long* __restrict__ start, long long F, long long r) {
  long long lo = 0, hi = F - 1;
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (start[mid] <= r) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct KRaster {
  const double* uv;
  const int* box;
  const long long* start;
  long long F, work;
  int N;
};

__device__ __forceinline__ void work_item(const KRaster& A, long long r, long long& f, int& col, int& row) {
  f = work_face(A.start, A.F, r);
  const unsigned q = (unsigned)(r - A.start[f]), w = (unsigned)A.box[4 * f + 2];  // a box holds at most N^2 < 2^31 texels
  const unsigned y = q / w;
  col = A.box[4 * f] + (int)(q - y * w);
  row = A.box[4 * f + 1] + (int)y;
}

__global__ void __launch_bounds__(kThreads) conflict_kernel(KRaster A, int* cnt, int* minf) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < A.work; r += (long long)gridDim.x * blockDim.x) {
    long long f;
    int col, row;
    work_item(A, r, f, col, row);
    Tri t;
    load_tri(A.uv, f, t);
    if (strictly_inside(t, col + 0.5, row + 0.5)) {
      const size_t tx = (size_t)row * A.N + col;
      atomicAdd(cnt + tx, 1);
      atomicMin(minf + tx, (int)f);
    }
  }
}

__global__ void __launch_bounds__(kThreads) mark_kernel(KRaster A, const int* __restrict__ cnt, const int* __restrict__ minf, int* cut,
                                                        int* added) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < A.work; r += (long long)gridDim.x * blockDim.x) {
    long long f;
    int col, row;
    work_item(A, r, f, col, row);
    const size_t tx = (size_t)row * A.N + col;
    if (cnt[tx] < 2 || minf[tx] == (int)f) continue;
    Tri t;
    load_tri(A.uv, f, t);
    if (strictly_inside(t, col + 0.5, row + 0.5) && atomicExch(cut + f, 1) == 0) atomicAdd(added, 1);
  }
}

__global__ void __launch_bounds__(kThreads) owner_kernel(KRaster A, unsigned long long* keys) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < A.work; r += (long long)gridDim.x * blockDim.x) {
    long long f;
    int col, row;
    work_item(A, r, f, col, row);
    Tri t;
    load_tri(A.uv, f, t);
    float w0, w1, w2;
    const double d2 = closest(t, col + 0.5, row + 0.5, w0, w1, w2);
    if (d2 <= kGutter * kGutter) {
      const unsigned long long key = ((unsigned long long)__float_as_uint(__double2float_rn(d2)) << 32) | (unsigned long long)f;
      atomicMin(keys + (size_t)row * A.N + col, key);
    }
  }
}

__global__ void __launch_bounds__(kThreads) owned_kernel(const unsigned long long* __restrict__ keys, long long n, int* __restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) flag[i] = keys[i] != kNoOwner;
}

__global__ void __launch_bounds__(kThreads) compact_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ at, const double* __restrict__ uv,
                                                           long long n, int N, int32_t* __restrict__ owner, int32_t* __restrict__ texels,
                                                           int32_t* __restrict__ texel_faces, float* __restrict__ bary) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (k == kNoOwner) {
      owner[i] = -1;
      continue;
    }
    const int f = (int)(k & 0xFFFFFFFFull), j = at[i];
    owner[i] = f;
    texels[j] = (int)i;
    texel_faces[j] = f;
    Tri t;
    load_tri(uv, f, t);
    float w0, w1, w2;
    closest(t, (int)(i % N) + 0.5, (int)(i / N) + 0.5, w0, w1, w2);
    bary[3 * (size_t)j] = w0;
    bary[3 * (size_t)j + 1] = w1;
    bary[3 * (size_t)j + 2] = w2;
  }
}

struct UScratch {
  double *proj, *ext, *pmin;                   // [6F], [2F], [2F]
  unsigned long long *keys_in, *keys, *lo, *hi;  // [3F], [3F], [2F], [2F]
  int *vals_in, *vals;                          // [3F]
  int *parent, *flag, *rank, *cut, *box;        // [F] x4, [4F]
  long long *boxn, *start;                      // [F]
  unsigned long long* tkeys;                    // [N^2]; cnt / minf of the conflict raster alias it
  int *oflag, *oat;                             // [N^2]
  int* counters;                                // bad, charts, added singletons, owned
  void* cub;
  size_t cub_bytes;
};

int unwrap_cub_bytes(long long F, long long NN, size_t* bytes) {
  size_t a = 0, b = 0, c = 0;
  const int ne = (int)std::max(3 * F, 1LL);
  if (check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, a, (const int*)nullptr, (int*)nullptr, (int)std::max(F, NN)), "cub ExclusiveSum size query") ||
      check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, b, (const long long*)nullptr, (long long*)nullptr, (int)std::max(F, 1LL)),
                 "cub ExclusiveSum size query") ||
      check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, c, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const int*)nullptr,
                                                 (int*)nullptr, ne),
                 "cub SortPairs size query"))
    return FNR_ERR_CUDA;
  *bytes = std::max(a, std::max(b, c));
  return FNR_OK;
}

size_t ucarve(char* base, long long F, long long NN, size_t cub_size, UScratch* s) {
  size_t off = 0;
  const size_t f = (size_t)std::max(F, 1LL), e = 3 * f, t = (size_t)NN;
  auto take = [&](size_t bytes) -> char* {
    char* p = base ? base + off : nullptr;
    off += (bytes + 255) / 256 * 256;
    return p;
  };
  s->proj = (double*)take(48 * f);
  s->ext = (double*)take(16 * f);
  s->pmin = (double*)take(16 * f);
  s->keys_in = (unsigned long long*)take(8 * e);
  s->keys = (unsigned long long*)take(8 * e);
  s->lo = (unsigned long long*)take(16 * f);
  s->hi = (unsigned long long*)take(16 * f);
  s->vals_in = (int*)take(4 * e);
  s->vals = (int*)take(4 * e);
  s->parent = (int*)take(4 * f);
  s->flag = (int*)take(4 * f);
  s->rank = (int*)take(4 * f);
  s->cut = (int*)take(4 * f);
  s->box = (int*)take(16 * f);
  s->boxn = (long long*)take(8 * f);
  s->start = (long long*)take(8 * f);
  s->tkeys = (unsigned long long*)take(8 * t);
  s->oflag = (int*)take(4 * t);
  s->oat = (int*)take(4 * t);
  s->counters = (int*)take(16);
  s->cub = take(cub_size);
  s->cub_bytes = cub_size;
  return off;
}

int blocks(long long work) { return grid_for(std::max(work, 1LL), kThreads, sm_count() * 32); }

#define FNR_LAUNCH(kernel, work, ...)                                          \
  do {                                                                         \
    kernel<<<blocks(work), kThreads, 0, st>>>(__VA_ARGS__);                    \
    if (int rc_ = check_launch(#kernel)) return rc_;                           \
  } while (0)

#define FNR_CUDA(call, what)                                                   \
  do {                                                                         \
    if (int rc_ = check_cuda((call), what)) return rc_;                        \
  } while (0)

int check_unwrap_args(const char* what, int64_t V, int64_t F, int32_t N) {
  if (V < 1 || F < 1 || N < FNR_UNWRAP_MIN_SIDE || N > FNR_TEXTURE_MAX_SIDE) {
    set_error("%s: needs V >= 1, F >= 1 and %d <= num_pixels_per_side <= %d, got %lld vertices, %lld faces, %d", what, FNR_UNWRAP_MIN_SIDE,
              FNR_TEXTURE_MAX_SIDE, (long long)V, (long long)F, N);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (V > kMaxIndex || F > kMaxFaces) {
    set_error("%s: %lld vertices or %lld faces exceed 2^31 - 1 vertices or (2^31 - 1) / 3 faces", what, (long long)V, (long long)F);
    return FNR_ERR_UNSUPPORTED;
  }
  return FNR_OK;
}

double elapsed_ms(std::chrono::steady_clock::time_point& t0) {
  const auto t1 = std::chrono::steady_clock::now();
  const double ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  t0 = t1;
  return ms;
}

}  // namespace

// Next-fit shelves of the charts, taken in `order`, at scale s into N x N; false when one does not fit.
static bool unwrap_pack(const double* ext, const std::vector<int>& order, double s, int N, int32_t* offsets) {
  long long x = 0, y = 0, shelf = 0;
  for (const int c : order) {
    const long long w = (long long)std::floor(s * ext[2 * c]) + 1 + 2 * kMargin, h = (long long)std::floor(s * ext[2 * c + 1]) + 1 + 2 * kMargin;
    if (w > N) return false;
    if (x + w > N) {
      y += shelf;
      x = 0;
      shelf = 0;
    }
    if (y + h > N) return false;
    offsets[2 * c] = (int32_t)x;
    offsets[2 * c + 1] = (int32_t)y;
    x += w;
    shelf = std::max(shelf, h);
  }
  return true;
}

// The largest scale that packs after FNR_UNWRAP_BISECTIONS fp64 halvings of [0, N / largest extent], and its offsets;
// -1 when the charts do not fit even at scale 0 (7 x 7 texels each).
static double unwrap_scale(const double* ext, long long C, int N, int32_t* offsets) {
  std::vector<int> order(C);
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](int a, int b) {
    if (ext[2 * a + 1] != ext[2 * b + 1]) return ext[2 * a + 1] > ext[2 * b + 1];
    if (ext[2 * a] != ext[2 * b]) return ext[2 * a] > ext[2 * b];
    return a < b;
  });
  if (!unwrap_pack(ext, order, 0.0, N, offsets)) return -1.0;
  double emax = 0.0;
  for (long long i = 0; i < 2 * C; ++i) emax = std::max(emax, ext[i]);
  if (!(emax > 0.0)) return 0.0;
  double lo = 0.0, hi = (double)N / emax;
  for (int k = 0; k < FNR_UNWRAP_BISECTIONS; ++k) {
    const double mid = (lo + hi) * 0.5;
    if (unwrap_pack(ext, order, mid, N, offsets)) lo = mid;
    else hi = mid;
  }
  unwrap_pack(ext, order, lo, N, offsets);
  return lo;
}

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_chart_unwrap_scratch_bytes(int64_t num_vertices, int64_t num_faces, int32_t num_pixels_per_side, size_t* bytes) {
  const char* what = "fnr_chart_unwrap_scratch_bytes";
  if (!bytes) {
    set_error("%s: NULL bytes", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_unwrap_args(what, num_vertices, num_faces, num_pixels_per_side)) return rc;
  const long long NN = (long long)num_pixels_per_side * num_pixels_per_side;
  size_t cb = 0;
  if (int rc = unwrap_cub_bytes(num_faces, NN, &cb)) return rc;
  UScratch s;
  *bytes = ucarve(nullptr, num_faces, NN, cb, &s);
  return FNR_OK;
}

int fnr_chart_unwrap(const float* vertices, const int64_t* faces, int64_t num_vertices, int64_t num_faces, int32_t num_pixels_per_side,
                     void* scratch, size_t scratch_bytes, int32_t* labels, int32_t* charts, int32_t* offsets, double* uv, int32_t* owner,
                     int32_t* texels, int32_t* texel_faces, float* barycentrics, int32_t* out_rounds, int64_t* out_num_charts,
                     double* out_scale, int64_t* out_num_owned, double* stage_ms, void* stream) {
  const char* what = "fnr_chart_unwrap";
  if (!vertices || !faces || !scratch || !labels || !charts || !offsets || !uv || !owner || !texels || !texel_faces || !barycentrics || !out_rounds ||
      !out_num_charts || !out_scale || !out_num_owned) {
    set_error("%s: NULL pointer", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_unwrap_args(what, num_vertices, num_faces, num_pixels_per_side)) return rc;
  const int N = num_pixels_per_side;
  const long long F = num_faces, V = num_vertices, NN = (long long)N * N, E = 3 * F;
  size_t cb = 0;
  if (int rc = unwrap_cub_bytes(F, NN, &cb)) return rc;
  UScratch s;
  const size_t need = ucarve(nullptr, F, NN, cb, &s);
  if (scratch_bytes < need) {
    set_error("%s: scratch too small: need %zu bytes, got %zu", what, need, scratch_bytes);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  ucarve(static_cast<char*>(scratch), F, NN, cb, &s);
  *out_rounds = 0;
  *out_num_charts = 0;
  *out_scale = -1.0;
  *out_num_owned = 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto t0 = std::chrono::steady_clock::now();
  double ms[FNR_UNWRAP_STAGES] = {0, 0, 0, 0, 0};
  auto stage = [&](int k) -> int {  // with timing, the stream is drained at each stage boundary
    if (!stage_ms) return FNR_OK;
    if (int rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize")) return rc;
    ms[k] += elapsed_ms(t0);
    return FNR_OK;
  };
  int host[4] = {0, 0, 0, 0};
  // labels, projections and the sorted half-edges, once
  FNR_CUDA(cudaMemsetAsync(s.counters, 0, 4 * sizeof(int), st), "cudaMemsetAsync");
  FNR_CUDA(cudaMemsetAsync(s.cut, 0, sizeof(int) * (size_t)F, st), "cudaMemsetAsync");
  FNR_LAUNCH(prepare_kernel, F, KPrepare{vertices, faces, V, F, labels, s.proj, s.keys_in, s.vals_in, s.counters});
  size_t tb = s.cub_bytes;
  FNR_CUDA(sort_half_edges(s.cub, tb, s.keys_in, s.keys, s.vals_in, s.vals, E, V, st), "cub SortPairs (half-edges)");
  FNR_CUDA(cudaMemcpyAsync(host, s.counters, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
  FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
  if (host[0]) {
    set_error("%s: a face index lies outside [0, %lld) or a vertex of a face is not finite", what, V);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = stage(0)) return rc;
  std::vector<double> ext;
  std::vector<int32_t> off;
  double scale = 0.0;
  long long C = 0, work = 0;
  int rounds = 0;
  for (;;) {
    // charts: union-find over the interior edges, numbered by their smallest face
    FNR_LAUNCH(iota_kernel, F, s.parent, F);
    FNR_LAUNCH(link_kernel, E, s.keys, s.vals, E, labels, s.cut, s.parent);
    FNR_LAUNCH(flatten_kernel, F, s.parent, s.flag, F);
    tb = s.cub_bytes;
    FNR_CUDA(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.flag, s.rank, (int)F, st), "cub ExclusiveSum (charts)");
    FNR_LAUNCH(chart_kernel, F, s.parent, s.rank, F, charts, s.lo, s.hi);
    FNR_LAUNCH(extent_kernel, F, s.proj, charts, F, s.lo, s.hi);
    int last[2] = {0, 0};
    FNR_CUDA(cudaMemcpyAsync(last, s.rank + F - 1, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaMemcpyAsync(last + 1, s.flag + F - 1, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    C = (long long)last[0] + last[1];
    FNR_LAUNCH(extent_finish_kernel, 2 * C, s.lo, s.hi, C, s.ext, s.pmin);
    ext.resize(2 * C);
    off.resize(2 * C);
    FNR_CUDA(cudaMemcpyAsync(ext.data(), s.ext, sizeof(double) * 2 * (size_t)C, cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (int rc = stage(1)) return rc;
    // packing on the host
    scale = unwrap_scale(ext.data(), C, N, off.data());
    *out_rounds = rounds;
    *out_num_charts = C;
    if (scale < 0.0) {
      if (stage_ms) std::copy(ms, ms + FNR_UNWRAP_STAGES, stage_ms);
      return FNR_OK;  // does not fit: *out_scale stays -1
    }
    FNR_CUDA(cudaMemcpyAsync(offsets, off.data(), sizeof(int32_t) * 2 * (size_t)C, cudaMemcpyHostToDevice, st), "cudaMemcpyAsync");
    if (int rc = stage(2)) return rc;
    // raster: texel coordinates, boxes, conflicts
    FNR_LAUNCH(uv_kernel, F, s.proj, charts, offsets, s.pmin, scale, F, N, uv, s.box, s.boxn);
    tb = s.cub_bytes;
    FNR_CUDA(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.boxn, s.start, (int)F, st), "cub ExclusiveSum (boxes)");
    long long lastw[2] = {0, 0};
    FNR_CUDA(cudaMemcpyAsync(lastw, s.start + F - 1, sizeof(long long), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaMemcpyAsync(lastw + 1, s.boxn + F - 1, sizeof(long long), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    work = lastw[0] + lastw[1];
    const KRaster R{uv, s.box, s.start, F, work, N};
    int* cnt = reinterpret_cast<int*>(s.tkeys);
    int* minf = cnt + NN;
    FNR_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int) * (size_t)NN, st), "cudaMemsetAsync");
    FNR_CUDA(cudaMemsetAsync(minf, 0x7F, sizeof(int) * (size_t)NN, st), "cudaMemsetAsync");
    FNR_CUDA(cudaMemsetAsync(s.counters + 2, 0, sizeof(int), st), "cudaMemsetAsync");
    FNR_LAUNCH(conflict_kernel, work, R, cnt, minf);
    FNR_LAUNCH(mark_kernel, work, R, cnt, minf, s.cut, s.counters + 2);
    FNR_CUDA(cudaMemcpyAsync(host + 2, s.counters + 2, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (int rc = stage(3)) return rc;
    if (host[2] == 0) break;
    ++rounds;
  }
  // owners within the gutter, compacted in texel order with their barycentrics
  const KRaster R{uv, s.box, s.start, F, work, N};
  FNR_CUDA(cudaMemsetAsync(s.tkeys, 0xFF, sizeof(unsigned long long) * (size_t)NN, st), "cudaMemsetAsync");
  FNR_LAUNCH(owner_kernel, work, R, s.tkeys);
  FNR_LAUNCH(owned_kernel, NN, s.tkeys, NN, s.oflag);
  tb = s.cub_bytes;
  FNR_CUDA(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.oflag, s.oat, (int)NN, st), "cub ExclusiveSum (owned texels)");
  FNR_LAUNCH(compact_kernel, NN, s.tkeys, s.oat, uv, NN, N, owner, texels, texel_faces, barycentrics);
  int lasto[2] = {0, 0};
  FNR_CUDA(cudaMemcpyAsync(lasto, s.oat + NN - 1, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
  FNR_CUDA(cudaMemcpyAsync(lasto + 1, s.oflag + NN - 1, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
  FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
  if (int rc = stage(4)) return rc;
  *out_rounds = rounds;
  *out_num_charts = C;
  *out_scale = scale;
  *out_num_owned = (long long)lasto[0] + lasto[1];
  if (stage_ms) std::copy(ms, ms + FNR_UNWRAP_STAGES, stage_ms);
  return FNR_OK;
}

}  // extern "C"
