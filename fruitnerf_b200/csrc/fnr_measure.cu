// Per-fruit measurement of triangle meshes (`python -m fruitnerf_b200.scripts.measure`; DESIGN section 4.3n).  Each face
// carries a group label; every quantity is computed per group.
//   check_faces_kernel     refuses face indices outside [0, V), labels outside [-1, G) and non-finite centres (one device
//                          flag, one host read, before any kernel reads through a face index)
//   uf_hook_kernel         connected components through shared vertex indices: union-find whose roots hook to the smaller
//   uf_flatten_kernel      root with atomicCAS, then pointer jumping.  A root is its component's smallest vertex, so
//   face_label_kernel      renumbering the used roots by an exclusive scan orders the groups by smallest vertex index
//   assign_kernel          centre mode: each face goes to the nearest centre of its centroid (centres tiled through
//                          shared memory; fp64 squared distance with no FMA; ties to the lower index)
//   edge_classify_kernel   the 3F half-edges radix-sorted by their (min, max) vertex key: per run of equal keys and per
//                          group in it, one half-edge is a boundary edge, two an interior edge, three or more a
//                          non-manifold edge (integer atomics)
//   group_kernel           one block per group over its faces in input order (the faces stably radix-sorted by group):
//                          pass 1 area and area-weighted centroid, pass 2 the moments of the area-weighted algebraic
//                          (Kasa) sphere fit solved by one thread with partial pivoting, pass 3 the RMS of the fit, the
//                          star volume and the solid angle (Van Oosterom-Strackee) about the fitted centre
// Every fp64 operation is rounded where written (__dadd_rn, __dmul_rn, ...), and each block combines its partial sums in
// a fixed order, so repeated calls give identical bits and measure.py restates the kernels.
#include <cub/cub.cuh>
#include <algorithm>
#include <climits>
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_kernels.h"
#include "fnr_mesh_edges.cuh"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr long long kMaxIndex = 2147483647LL;
constexpr long long kMaxFaces = kMaxIndex / 3;  // the half-edges are sorted as one cub call of int-sized length
constexpr double kPivotTol = 1e-12;             // |pivot| of the normalised 4x4 system at or below which the fit fails

enum BadFlag { kBadIndex = 1, kBadLabel = 2, kBadCenter = 4 };

__global__ void __launch_bounds__(kThreads) check_faces_kernel(const int64_t* __restrict__ faces, long long F, long long V,
                                                               const int32_t* __restrict__ labels, long long G,
                                                               const double* __restrict__ centers, long long K, int* __restrict__ bad) {
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < 3 * K; c += (long long)gridDim.x * blockDim.x)
    if (!isfinite(centers[c])) atomicOr(bad, kBadCenter);
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    int b = 0;
    for (int k = 0; k < 3; ++k) {
      const long long v = faces[3 * f + k];
      if (v < 0 || v >= V) b |= kBadIndex;
    }
    if (labels && (labels[f] < -1 || labels[f] >= G)) b |= kBadLabel;
    if (b) atomicOr(bad, b);
  }
}

// ---- connected components ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) uf_init_kernel(int* __restrict__ parent, int* __restrict__ used, long long V) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    parent[v] = (int)v;
    used[v] = 0;
  }
}

// Root of x with path halving.  parent[v] <= v always holds, so every store writes an ancestor and races are benign.
__device__ __forceinline__ int uf_find(int* parent, int x) {
  volatile int* p = parent;
  int cur = p[x];
  if (cur != x) {
    int prev = x, next;
    while (cur > (next = p[cur])) {
      p[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

__device__ __forceinline__ void uf_unite(int* parent, int a, int b) {
  int ra = uf_find(parent, a), rb = uf_find(parent, b);
  while (ra != rb) {
    const int hi = ra > rb ? ra : rb, lo = ra > rb ? rb : ra;
    const int old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) return;
    // hi was hooked meanwhile: continue from where it now points
    ra = uf_find(parent, old);
    rb = uf_find(parent, lo);
  }
}

__global__ void __launch_bounds__(kThreads) uf_hook_kernel(const int64_t* __restrict__ faces, long long F, int* parent,
                                                           int* __restrict__ used) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    const int a = (int)faces[3 * f], b = (int)faces[3 * f + 1], c = (int)faces[3 * f + 2];
    used[a] = 1;
    used[b] = 1;
    used[c] = 1;
    uf_unite(parent, a, b);
    uf_unite(parent, b, c);
  }
}

// parent[v] = root; used[v] becomes "v is the root of a component that has faces".  The walk to the root writes nothing:
// a path-halving store of another thread could otherwise replace a root just written with a stale, non-root ancestor.
__global__ void __launch_bounds__(kThreads) uf_flatten_kernel(int* parent, int* __restrict__ used, long long V) {
  volatile int* p = parent;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    int r = p[v], next;
    while (r != (next = p[r])) r = next;
    p[v] = r;
    used[v] = (used[v] && r == (int)v) ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kThreads) face_label_kernel(const int64_t* __restrict__ faces, long long F, const int* __restrict__ parent,
                                                              const int* __restrict__ ids, int32_t* __restrict__ face_group) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x)
    face_group[f] = ids[parent[faces[3 * f]]];
}

__global__ void group_total_kernel(const int* __restrict__ flag, const int* __restrict__ ids, long long V, int* __restrict__ total) {
  *total = ids[V - 1] + flag[V - 1];
}

// ---- centre assignment ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void face_vertices(const double* __restrict__ verts, const int64_t* __restrict__ faces, long long f, double v[3][3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const long long i = __ldg(faces + 3 * f + k);
#pragma unroll
    for (int a = 0; a < 3; ++a) v[k][a] = __ldg(verts + 3 * i + a);
  }
}

// (v0 + v1 + v2) / 3, summed left to right
__device__ __forceinline__ void face_centroid(const double v[3][3], double c[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = __ddiv_rn(__dadd_rn(__dadd_rn(v[0][a], v[1][a]), v[2][a]), 3.0);
}

__global__ void __launch_bounds__(kThreads) assign_kernel(const double* __restrict__ verts, const int64_t* __restrict__ faces, long long F,
                                                          const double* __restrict__ centers, int K, double max_d2, int32_t* __restrict__ out) {
  __shared__ double s_c[3 * kThreads];
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double c[3] = {0.0, 0.0, 0.0};
  if (f < F) {
    double v[3][3];
    face_vertices(verts, faces, f, v);
    face_centroid(v, c);
  }
  double best = CUDART_INF;
  int bi = -1;
  for (int t0 = 0; t0 < K; t0 += kThreads) {
    const int m = min(kThreads, K - t0);
    __syncthreads();
    if (threadIdx.x < m)
      for (int a = 0; a < 3; ++a) s_c[3 * threadIdx.x + a] = centers[3 * (size_t)(t0 + threadIdx.x) + a];
    __syncthreads();
    for (int j = 0; j < m; ++j) {
      const double d = dist2(c[0], c[1], c[2], s_c[3 * j], s_c[3 * j + 1], s_c[3 * j + 2]);
      if (d < best) {
        best = d;
        bi = t0 + j;
      }
    }
  }
  if (f < F) out[f] = (bi >= 0 && best <= max_d2) ? bi : -1;
}

// ---- edges ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) sort_inputs_kernel(const int64_t* __restrict__ faces, long long F, long long V,
                                                               const int32_t* __restrict__ labels, uint32_t* __restrict__ gkeys,
                                                               int* __restrict__ fidx, unsigned long long* __restrict__ ekeys,
                                                               int* __restrict__ egroup) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    const int g = labels[f];
    gkeys[f] = (uint32_t)(g + 1);  // unassigned faces (-1) sort first
    fidx[f] = (int)f;
    for (int k = 0; k < 3; ++k) {
      ekeys[3 * f + k] = half_edge_key((unsigned long long)faces[3 * f + k], (unsigned long long)faces[3 * f + (k + 1) % 3], (unsigned long long)V);
      egroup[3 * f + k] = g;
    }
  }
}

__global__ void __launch_bounds__(kThreads) edge_classify_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ group,
                                                                 long long E, unsigned long long* __restrict__ boundary,
                                                                 unsigned long long* __restrict__ nonmanifold) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (i > 0 && keys[i - 1] == k) continue;  // one thread per run of equal keys
    long long end = i + 1;
    while (end < E && keys[end] == k) ++end;
    for (long long j = i; j < end; ++j) {
      const int g = group[j];
      if (g < 0) continue;
      bool first = true;
      for (long long q = i; q < j && first; ++q) first = group[q] != g;
      if (!first) continue;
      int c = 1;
      for (long long q = j + 1; q < end; ++q) c += group[q] == g;
      if (c == 1) atomicAdd(boundary + g, 1ull);
      else if (c >= 3) atomicAdd(nonmanifold + g, 1ull);
    }
  }
}

// ---- per-group sums ---------------------------------------------------------------------------------------------------
// Sum over the block of K values per thread, in a fixed order (warp tree, then the warps in order); every thread gets
// the sums.
template <int K>
__device__ __forceinline__ void block_sums(double (&v)[K], double (*s)[kWarps]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double x = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = __dadd_rn(x, __shfl_down_sync(0xffffffffu, x, o));
    if (lane == 0) s[k][warp] = x;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double r = 0.0;
    for (int w = 0; w < kWarps; ++w) r = __dadd_rn(r, s[k][w]);
    v[k] = r;
  }
  __syncthreads();
}

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double c[3]) {
  c[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  c[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  c[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}

__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

// |e1 x e2| / 2
__device__ __forceinline__ double face_area(const double v[3][3]) {
  double e1[3], e2[3], n[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    e1[a] = __dsub_rn(v[1][a], v[0][a]);
    e2[a] = __dsub_rn(v[2][a], v[0][a]);
  }
  cross3(e1, e2, n);
  return __dmul_rn(__dsqrt_rn(dot3(n, n)), 0.5);
}

__device__ __forceinline__ long long lower_bound_u32(const uint32_t* __restrict__ a, long long n, uint32_t key) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// The Kasa fit about the centroid from the area-weighted moments (A = sum w, S = sum w p p^T, s1 = sum w p, t = sum w p |p|^2,
// T = sum w |p|^2).  Coordinates are scaled by sc = sqrt(T / A) and the system by 1 / A, then solved by Gaussian
// elimination with partial pivoting.  Returns false (fit failed) on a pivot <= kPivotTol or d + |x|^2 <= 0; x, r on success.
__device__ bool kasa_solve(double A, const double S[6], const double s1[3], const double t[3], double T, double x[3], double& r) {
  if (!(A > 0.0)) return false;
  const double s2 = __ddiv_rn(T, A);
  if (!(s2 > 0.0)) return false;
  const double sc = __dsqrt_rn(s2);
  const double as2 = __dmul_rn(A, s2), as1 = __dmul_rn(A, sc), as3 = __dmul_rn(as2, sc);
  const int ij[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};  // S = xx, xy, xz, yy, yz, zz
  double M[4][5];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) M[i][j] = __ddiv_rn(__dmul_rn(4.0, S[ij[i][j]]), as2);
    M[i][3] = __ddiv_rn(__dmul_rn(2.0, s1[i]), as1);
    M[3][i] = M[i][3];
    M[i][4] = __ddiv_rn(__dmul_rn(2.0, t[i]), as3);
  }
  M[3][3] = 1.0;
  M[3][4] = __ddiv_rn(T, as2);
  for (int k = 0; k < 4; ++k) {
    int p = k;
    for (int i = k + 1; i < 4; ++i)
      if (fabs(M[i][k]) > fabs(M[p][k])) p = i;
    if (!(fabs(M[p][k]) > kPivotTol)) return false;
    if (p != k)
      for (int j = 0; j < 5; ++j) {
        const double tmp = M[k][j];
        M[k][j] = M[p][j];
        M[p][j] = tmp;
      }
    for (int i = k + 1; i < 4; ++i) {
      const double f = __ddiv_rn(M[i][k], M[k][k]);
      for (int j = k; j < 5; ++j) M[i][j] = __dsub_rn(M[i][j], __dmul_rn(f, M[k][j]));
    }
  }
  double u[4];
  for (int k = 3; k >= 0; --k) {
    double acc = M[k][4];
    for (int j = k + 1; j < 4; ++j) acc = __dsub_rn(acc, __dmul_rn(M[k][j], u[j]));
    u[k] = __ddiv_rn(acc, M[k][k]);
  }
  const double rr = __dadd_rn(u[3], __dadd_rn(__dadd_rn(__dmul_rn(u[0], u[0]), __dmul_rn(u[1], u[1])), __dmul_rn(u[2], u[2])));
  if (!(rr > 0.0)) return false;
  for (int a = 0; a < 3; ++a) x[a] = __dmul_rn(u[a], sc);
  r = __dmul_rn(__dsqrt_rn(rr), sc);
  return true;
}

struct KGroups {
  const double* verts;
  const int64_t* faces;
  long long F;
  const uint32_t* gkeys;  // sorted labels + 1
  const int* perm;        // face of each sorted position
  long long G;
  long long* group_faces;
  double *area, *centroid, *sphere, *volume, *coverage;
  int32_t* fit_ok;
  long long* unassigned_faces;
  double* unassigned_area;
};

__global__ void __launch_bounds__(kThreads) group_kernel(KGroups A) {
  __shared__ double s_red[13][kWarps];
  __shared__ double s_fit[5];  // centre xyz, r, fit_ok
  const long long g = blockIdx.x;
  const uint32_t key = g < A.G ? (uint32_t)(g + 1) : 0u;  // the last block takes the unassigned faces
  const long long lo = lower_bound_u32(A.gkeys, A.F, key), hi = lower_bound_u32(A.gkeys, A.F, key + 1);
  const long long n = hi - lo;
  // pass 1: area, area-weighted and plain centroid sums
  double s[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long j = lo + threadIdx.x; j < hi; j += kThreads) {
    double v[3][3], c[3];
    face_vertices(A.verts, A.faces, A.perm[j], v);
    face_centroid(v, c);
    const double w = face_area(v);
    s[0] = __dadd_rn(s[0], w);
    for (int a = 0; a < 3; ++a) {
      s[1 + a] = __dadd_rn(s[1 + a], __dmul_rn(w, c[a]));
      s[4 + a] = __dadd_rn(s[4 + a], c[a]);
    }
  }
  block_sums<7>(s, s_red);
  const double area = s[0];
  if (key == 0) {
    if (threadIdx.x == 0) {
      *A.unassigned_faces = n;
      *A.unassigned_area = area;
    }
    return;
  }
  const double nan = CUDART_NAN;
  if (n == 0) {
    if (threadIdx.x == 0) {
      A.group_faces[g] = 0;
      A.area[g] = 0.0;
      for (int a = 0; a < 3; ++a) A.centroid[3 * g + a] = nan;
      for (int a = 0; a < 5; ++a) A.sphere[5 * g + a] = nan;
      A.volume[g] = 0.0;
      A.coverage[g] = 0.0;
      A.fit_ok[g] = 0;
    }
    return;
  }
  double m[3];
  for (int a = 0; a < 3; ++a) m[a] = area > 0.0 ? __ddiv_rn(s[1 + a], area) : __ddiv_rn(s[4 + a], (double)n);
  // pass 2: moments of the face centroids about m, weighted by area
  double q[13];
  for (int k = 0; k < 13; ++k) q[k] = 0.0;
  for (long long j = lo + threadIdx.x; j < hi; j += kThreads) {
    double v[3][3], c[3], p[3], wp[3];
    face_vertices(A.verts, A.faces, A.perm[j], v);
    face_centroid(v, c);
    const double w = face_area(v);
    for (int a = 0; a < 3; ++a) {
      p[a] = __dsub_rn(c[a], m[a]);
      wp[a] = __dmul_rn(w, p[a]);
    }
    const double pp = dot3(p, p);
    q[0] = __dadd_rn(q[0], __dmul_rn(wp[0], p[0]));
    q[1] = __dadd_rn(q[1], __dmul_rn(wp[0], p[1]));
    q[2] = __dadd_rn(q[2], __dmul_rn(wp[0], p[2]));
    q[3] = __dadd_rn(q[3], __dmul_rn(wp[1], p[1]));
    q[4] = __dadd_rn(q[4], __dmul_rn(wp[1], p[2]));
    q[5] = __dadd_rn(q[5], __dmul_rn(wp[2], p[2]));
    for (int a = 0; a < 3; ++a) {
      q[6 + a] = __dadd_rn(q[6 + a], wp[a]);
      q[9 + a] = __dadd_rn(q[9 + a], __dmul_rn(wp[a], pp));
    }
    q[12] = __dadd_rn(q[12], __dmul_rn(w, pp));
  }
  block_sums<13>(q, s_red);
  if (threadIdx.x == 0) {
    double x[3] = {0.0, 0.0, 0.0}, r = 0.0;
    const bool ok = kasa_solve(area, q, q + 6, q + 9, q[12], x, r);
    if (!ok) {  // the centroid, and the area-weighted RMS distance of the face centroids from it
      x[0] = x[1] = x[2] = 0.0;
      r = area > 0.0 ? __dsqrt_rn(__ddiv_rn(q[12], area)) : 0.0;
    }
    for (int a = 0; a < 3; ++a) s_fit[a] = __dadd_rn(m[a], x[a]);
    s_fit[3] = r;
    s_fit[4] = ok ? 1.0 : 0.0;
  }
  __syncthreads();
  const double ctr[3] = {s_fit[0], s_fit[1], s_fit[2]}, r = s_fit[3];
  // pass 3: fit residual, star volume and solid angle about ctr
  double t[3] = {0.0, 0.0, 0.0};
  for (long long j = lo + threadIdx.x; j < hi; j += kThreads) {
    double v[3][3], c[3], pc[3], d[3][3], bc[3];
    face_vertices(A.verts, A.faces, A.perm[j], v);
    face_centroid(v, c);
    const double w = face_area(v);
    for (int a = 0; a < 3; ++a) {
      pc[a] = __dsub_rn(c[a], ctr[a]);
      for (int k = 0; k < 3; ++k) d[k][a] = __dsub_rn(v[k][a], ctr[a]);
    }
    const double e = __dsub_rn(__dsqrt_rn(dot3(pc, pc)), r);
    t[0] = __dadd_rn(t[0], __dmul_rn(w, __dmul_rn(e, e)));
    cross3(d[1], d[2], bc);
    const double det = dot3(d[0], bc);
    t[1] = __dadd_rn(t[1], det);
    const double la = __dsqrt_rn(dot3(d[0], d[0])), lb = __dsqrt_rn(dot3(d[1], d[1])), lc = __dsqrt_rn(dot3(d[2], d[2]));
    const double den = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(la, lb), lc), __dmul_rn(dot3(d[0], d[1]), lc)),
                                           __dmul_rn(dot3(d[0], d[2]), lb)),
                                 __dmul_rn(dot3(d[1], d[2]), la));
    t[2] = __dadd_rn(t[2], __dmul_rn(2.0, atan2(det, den)));
  }
  block_sums<3>(t, s_red);
  if (threadIdx.x == 0) {
    A.group_faces[g] = n;
    A.area[g] = area;
    for (int a = 0; a < 3; ++a) {
      A.centroid[3 * g + a] = m[a];
      A.sphere[5 * g + a] = ctr[a];
    }
    A.sphere[5 * g + 3] = r;
    A.sphere[5 * g + 4] = area > 0.0 ? __dsqrt_rn(__ddiv_rn(t[0], area)) : 0.0;
    A.volume[g] = __ddiv_rn(t[1], 6.0);
    A.coverage[g] = __ddiv_rn(t[2], __dmul_rn(4.0, CUDART_PI));
    A.fit_ok[g] = s_fit[4] != 0.0;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
struct MScratch {
  int *parent, *flag, *ids;                  // [V]
  uint32_t *gkeys_in, *gkeys;                // [F]
  int *fidx_in, *perm;                       // [F]
  unsigned long long *ekeys_in, *ekeys;      // [3F]
  int *egroup_in, *egroup;                   // [3F]
  int* bad;
  int* total;
  void* cub;
  size_t cub_bytes;
};

int measure_cub_bytes(long long V, long long F, size_t* bytes) {
  size_t a = 0, b = 0, c = 0;
  const int nv = (int)std::max(V, 1LL), nf = (int)std::max(F, 1LL), ne = (int)std::max(3 * F, 1LL);
  if (check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, a, (const int*)nullptr, (int*)nullptr, nv), "cub ExclusiveSum size query") ||
      check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr, (int*)nullptr, nf),
                 "cub SortPairs (groups) size query") ||
      check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, c, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const int*)nullptr,
                                                 (int*)nullptr, ne),
                 "cub SortPairs (edges) size query"))
    return FNR_ERR_CUDA;
  *bytes = std::max(a, std::max(b, c));
  return FNR_OK;
}

size_t mcarve(char* base, long long V, long long F, size_t cub_size, MScratch* s) {
  size_t off = 0;
  const size_t v = (size_t)std::max(V, 1LL), f = (size_t)std::max(F, 1LL);
  auto take = [&](size_t bytes) -> char* {
    char* p = base ? base + off : nullptr;
    off += (bytes + 255) / 256 * 256;
    return p;
  };
  s->parent = (int*)take(4 * v);
  s->flag = (int*)take(4 * v);
  s->ids = (int*)take(4 * v);
  s->gkeys_in = (uint32_t*)take(4 * f);
  s->gkeys = (uint32_t*)take(4 * f);
  s->fidx_in = (int*)take(4 * f);
  s->perm = (int*)take(4 * f);
  s->ekeys_in = (unsigned long long*)take(24 * f);
  s->ekeys = (unsigned long long*)take(24 * f);
  s->egroup_in = (int*)take(12 * f);
  s->egroup = (int*)take(12 * f);
  s->bad = (int*)take(4);
  s->total = (int*)take(4);
  s->cub = take(cub_size);
  s->cub_bytes = cub_size;
  return off;
}

// V and F within what the kernels index with int: FNR_ERR_INVALID_ARGUMENT for negative counts, FNR_ERR_UNSUPPORTED above
int check_sizes(const char* what, int64_t V, int64_t F) {
  if (V < 0 || F < 0) {
    set_error("%s: negative counts (%lld vertices, %lld faces)", what, (long long)V, (long long)F);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (V > kMaxIndex || F > kMaxFaces) {
    set_error("%s: %lld vertices or %lld faces exceed 2^31 - 1 vertices or (2^31 - 1) / 3 faces", what, (long long)V, (long long)F);
    return FNR_ERR_UNSUPPORTED;
  }
  return FNR_OK;
}

int bind_mscratch(const char* what, long long V, long long F, void* scratch, size_t scratch_bytes, MScratch* s) {
  size_t cb = 0;
  if (int rc = measure_cub_bytes(V, F, &cb)) return rc;
  const size_t need = mcarve(nullptr, V, F, cb, s);
  if (!scratch || scratch_bytes < need) {
    set_error("%s: scratch too small: need %zu bytes, got %zu", what, need, scratch ? scratch_bytes : (size_t)0);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  mcarve(static_cast<char*>(scratch), V, F, cb, s);
  return FNR_OK;
}

int blocks(long long work) { return grid_for(work, kThreads, sm_count() * 32); }

// Refuses a face index outside [0, V), (labels != NULL) a label outside [-1, G) and (K > 0) a non-finite centre: one host
// read of a device flag.
int check_faces(const char* what, const int64_t* faces, long long F, long long V, const int32_t* labels, long long G, const double* centers,
                long long K, int* bad, cudaStream_t st) {
  if (F == 0 && K == 0) return FNR_OK;
  if (int rc = check_cuda(cudaMemsetAsync(bad, 0, sizeof(int), st), "cudaMemsetAsync")) return rc;
  check_faces_kernel<<<blocks(std::max(F, 3 * K)), kThreads, 0, st>>>(faces, F, V, labels, G, centers, K, bad);
  if (int rc = check_launch("check_faces_kernel")) return rc;
  int h = 0;
  if (int rc = check_cuda(cudaMemcpyAsync(&h, bad, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync")) return rc;
  if (int rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize")) return rc;
  if (h & kBadIndex) {
    set_error("%s: a face index lies outside [0, %lld)", what, V);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (h & kBadLabel) {
    set_error("%s: a face label lies outside [-1, %lld)", what, G);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (h & kBadCenter) {
    set_error("%s: a centre is not finite", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  return FNR_OK;
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_mesh_measure_scratch_bytes(int64_t num_vertices, int64_t num_faces, size_t* bytes) {
  const char* what = "fnr_mesh_measure_scratch_bytes";
  if (!bytes) {
    set_error("%s: NULL bytes", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_sizes(what, num_vertices, num_faces)) return rc;
  size_t cb = 0;
  if (int rc = measure_cub_bytes(num_vertices, num_faces, &cb)) return rc;
  MScratch s;
  *bytes = mcarve(nullptr, num_vertices, num_faces, cb, &s);
  return FNR_OK;
}

int fnr_mesh_components(const int64_t* faces, int64_t num_faces, int64_t num_vertices, void* scratch, size_t scratch_bytes, int32_t* face_group,
                        int64_t* num_groups, void* stream) {
  const char* what = "fnr_mesh_components";
  if ((num_faces > 0 && (!faces || !face_group)) || !num_groups) {
    set_error("%s: NULL arguments", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_sizes(what, num_vertices, num_faces)) return rc;
  *num_groups = 0;
  MScratch s;
  if (int rc = bind_mscratch(what, num_vertices, num_faces, scratch, scratch_bytes, &s)) return rc;
  if (num_faces == 0) return FNR_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long V = num_vertices, F = num_faces;
  if (int rc = check_faces(what, faces, F, V, nullptr, 0, nullptr, 0, s.bad, st)) return rc;
  uf_init_kernel<<<blocks(V), kThreads, 0, st>>>(s.parent, s.flag, V);
  if (int rc = check_launch("uf_init_kernel")) return rc;
  uf_hook_kernel<<<blocks(F), kThreads, 0, st>>>(faces, F, s.parent, s.flag);
  if (int rc = check_launch("uf_hook_kernel")) return rc;
  uf_flatten_kernel<<<blocks(V), kThreads, 0, st>>>(s.parent, s.flag, V);
  if (int rc = check_launch("uf_flatten_kernel")) return rc;
  size_t tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.flag, s.ids, (int)V, st), "cub ExclusiveSum (group ids)")) return rc;
  group_total_kernel<<<1, 1, 0, st>>>(s.flag, s.ids, V, s.total);
  if (int rc = check_launch("group_total_kernel")) return rc;
  face_label_kernel<<<blocks(F), kThreads, 0, st>>>(faces, F, s.parent, s.ids, face_group);
  if (int rc = check_launch("face_label_kernel")) return rc;
  int total = 0;
  if (int rc = check_cuda(cudaMemcpyAsync(&total, s.total, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync")) return rc;
  if (int rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize")) return rc;
  *num_groups = total;
  return FNR_OK;
}

int fnr_mesh_assign_centers(const double* vertices, const int64_t* faces, int64_t num_faces, int64_t num_vertices, const double* centers,
                            int64_t num_centers, double max_distance, void* scratch, size_t scratch_bytes, int32_t* face_group, void* stream) {
  const char* what = "fnr_mesh_assign_centers";
  if ((num_faces > 0 && (!vertices || !faces || !face_group)) || (num_centers > 0 && !centers) || !scratch ||
      scratch_bytes < FNR_MESH_ASSIGN_SCRATCH_BYTES) {
    set_error("%s: NULL arguments or fewer than %d scratch bytes", what, FNR_MESH_ASSIGN_SCRATCH_BYTES);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_centers < 0 || std::isnan(max_distance) || !(max_distance > 0.0)) {
    set_error("%s: invalid arguments (%lld centres, max_distance %g)", what, (long long)num_centers, max_distance);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_sizes(what, num_vertices, num_faces)) return rc;
  if (num_centers > kMaxIndex) {
    set_error("%s: %lld centres exceed 2^31 - 1 groups", what, (long long)num_centers);
    return FNR_ERR_UNSUPPORTED;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (int rc = check_faces(what, faces, num_faces, num_vertices, nullptr, 0, centers, num_centers, static_cast<int*>(scratch), st)) return rc;
  if (num_faces == 0) return FNR_OK;
  const double md2 = max_distance * max_distance;
  assign_kernel<<<(unsigned)((num_faces + kThreads - 1) / kThreads), kThreads, 0, st>>>(vertices, faces, num_faces, centers, (int)num_centers, md2,
                                                                                       face_group);
  return check_launch("assign_kernel");
}

int fnr_mesh_measure_groups(const double* vertices, const int64_t* faces, int64_t num_faces, int64_t num_vertices, const int32_t* face_group,
                            int64_t num_groups, void* scratch, size_t scratch_bytes, int64_t* group_faces, int64_t* boundary_edges,
                            int64_t* nonmanifold_edges, double* area, double* centroid, double* sphere, double* volume, double* coverage,
                            int32_t* fit_ok, int64_t* unassigned_faces, double* unassigned_area, void* stream) {
  const char* what = "fnr_mesh_measure_groups";
  if ((num_faces > 0 && (!vertices || !faces || !face_group)) ||
      (num_groups > 0 && (!group_faces || !boundary_edges || !nonmanifold_edges || !area || !centroid || !sphere || !volume || !coverage || !fit_ok)) ||
      !unassigned_faces != !unassigned_area) {
    set_error("%s: NULL arguments", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_sizes(what, num_vertices, num_faces)) return rc;
  if (num_groups < 0) {
    set_error("%s: negative group count %lld", what, (long long)num_groups);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_groups > kMaxIndex - 1) {
    set_error("%s: %lld groups exceed 2^31 - 2", what, (long long)num_groups);
    return FNR_ERR_UNSUPPORTED;
  }
  MScratch s;
  if (int rc = bind_mscratch(what, num_vertices, num_faces, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long V = num_vertices, F = num_faces, G = num_groups;
  if (int rc = check_faces(what, faces, F, V, face_group, G, nullptr, 0, s.bad, st)) return rc;
  if (G > 0) {
    if (int rc = check_cuda(cudaMemsetAsync(boundary_edges, 0, sizeof(int64_t) * (size_t)G, st), "cudaMemsetAsync")) return rc;
    if (int rc = check_cuda(cudaMemsetAsync(nonmanifold_edges, 0, sizeof(int64_t) * (size_t)G, st), "cudaMemsetAsync")) return rc;
  }
  if (F > 0) {
    sort_inputs_kernel<<<blocks(F), kThreads, 0, st>>>(faces, F, V, face_group, s.gkeys_in, s.fidx_in, s.ekeys_in, s.egroup_in);
    if (int rc = check_launch("sort_inputs_kernel")) return rc;
    size_t tb = s.cub_bytes;
    if (int rc = check_cuda(cub::DeviceRadixSort::SortPairs(s.cub, tb, s.gkeys_in, s.gkeys, s.fidx_in, s.perm, (int)F, 0, bits_for((unsigned long long)G + 1), st),
                            "cub SortPairs (groups)"))
      return rc;
    tb = s.cub_bytes;
    if (int rc = check_cuda(sort_half_edges(s.cub, tb, s.ekeys_in, s.ekeys, s.egroup_in, s.egroup, 3 * F, V, st), "cub SortPairs (edges)"))
      return rc;
    if (G > 0) {
      edge_classify_kernel<<<blocks(3 * F), kThreads, 0, st>>>(s.ekeys, s.egroup, 3 * F, (unsigned long long*)boundary_edges,
                                                               (unsigned long long*)nonmanifold_edges);
      if (int rc = check_launch("edge_classify_kernel")) return rc;
    }
  }
  const long long nb = G + (unassigned_faces ? 1 : 0);
  if (nb == 0) return FNR_OK;
  KGroups A{vertices, faces, F, s.gkeys, s.perm, G, (long long*)group_faces, area, centroid, sphere, volume, coverage, fit_ok,
            (long long*)unassigned_faces, unassigned_area};
  group_kernel<<<(unsigned)nb, kThreads, 0, st>>>(A);
  return check_launch("group_kernel");
}

}  // extern "C"
