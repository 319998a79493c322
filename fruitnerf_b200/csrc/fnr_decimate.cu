// Quadric edge-collapse decimation of triangle meshes (`--target-num-faces` of the tsdf / poisson exports; DESIGN
// section 4.3q).  Garland-Heckbert quadrics, collapsed in rounds of independent edges:
//   prepare_kernel         refuses face indices outside [0, V) (one device flag, one host read) and copies the faces to
//                          int32 and the vertices to the working positions
//   half_edges_kernel      per round, the 3F half-edge keys (fnr_mesh_edges.cuh, shared with fnr_measure.cu) and the
//   vstart_kernel          (vertex, corner) incidence, both stably radix-sorted; vstart[v] opens v's corners
//   quadric_kernel         once: each vertex sums its corners in face order (the face's area-weighted plane, then the
//                          constraint planes of its boundary half-edges); fp64, no atomics
//   boundary_kernel        per round, the vertices on a boundary edge
//   cost_kernel            per edge: the validity checks on the mesh as it stands, the placement (3x3 elimination with
//                          partial pivoting) and the cost, as a 64-bit sort key (cost bits, +inf bits when not valid)
//   rank / m1 / m2 kernels ranks from one stable sort of the keys; m1[v] the least rank at v (integer atomicMin), m2[v]
//                          the least m1 over v and its neighbours
//   select_kernel          an edge is selected when its rank is m2 at both ends; its face count goes to its rank's slot,
//                          and an exclusive scan gives the faces removed before it
//   collapse_kernel        the selected edges before the face count reaches target + 1: b -> a, a to the placement,
//                          Q_a += Q_b (selected edges share no face, so no two touch the same vertex)
//   remap / compact        faces through the remap, those with a repeated index dropped, the rest compacted in order
//   normals_kernel         at the end: the normalised sum of right-hand face normals per vertex, in face order
// Every fp64 operation is rounded where written (__dadd_rn, __dmul_rn, ...; no FMA), so decimate.py restates the
// kernels bit for bit.  The host reads two integers per round and allocates nothing: one caller-sized scratch.
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
constexpr long long kMaxIndex = 2147483647LL;
constexpr long long kMaxFaces = kMaxIndex / 3;  // 3F half-edges and corners are sorted as int-sized cub calls
constexpr double kBoundaryWeight = 100.0;       // boundary constraint plane weight per |e|^2
constexpr double kPivotRel = 1e-8;              // pivot at or below kPivotRel * max diagonal: the placement falls back
constexpr unsigned long long kNoCost = 0x7FF0000000000000ull;  // bits of +inf: after every clamped finite cost
// quadric storage: xx xy xz xw yy yz yw zz zw ww; slot(i, j) is entry (i, j) (constant once the loops unroll)
__host__ __device__ constexpr int slot(int i, int j) {
  return (i < j ? i : j) == 0 ? (i < j ? j : i) : (i < j ? i : j) == 1 ? 3 + (i < j ? j : i) : (i < j ? i : j) == 2 ? 5 + (i < j ? j : i) : 9;
}

__device__ __forceinline__ void sub3(const double a[3], const double b[3], double c[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) c[k] = __dsub_rn(a[k], b[k]);
}

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double c[3]) {
  c[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  c[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  c[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}

__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

__device__ __forceinline__ void load3(const double* P, int v, double p[3]) {
  p[0] = P[3 * (size_t)v];
  p[1] = P[3 * (size_t)v + 1];
  p[2] = P[3 * (size_t)v + 2];
}

// (p1 - p0) x (p2 - p0)
__device__ __forceinline__ void face_normal(const double p0[3], const double p1[3], const double p2[3], double n[3]) {
  double e1[3], e2[3];
  sub3(p1, p0, e1);
  sub3(p2, p0, e2);
  cross3(e1, e2, n);
}

// q += w * p p^T of the plane with normal m through x (nothing when |m| = 0), entry by entry as w * (p_i * p_j)
__device__ __forceinline__ void add_plane(double q[10], const double m[3], const double x[3], double w) {
  const double ln = __dsqrt_rn(dot3(m, m));
  if (!(ln > 0.0)) {  // the plane's quadric is 0, and q + 0 = q
#pragma unroll
    for (int t = 0; t < 10; ++t) q[t] = __dadd_rn(q[t], 0.0);
    return;
  }
  double p[4];
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = __ddiv_rn(m[k], ln);
  p[3] = -dot3(p, x);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j) q[slot(i, j)] = __dadd_rn(q[slot(i, j)], __dmul_rn(w, __dmul_rn(p[i], p[j])));
}

// v^T Q v at v = (x, 1), clamped at 0
__device__ __forceinline__ double quadric_cost(const double q[10], const double x[3]) {
  double r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    r[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[slot(i, 0)], x[0]), __dmul_rn(q[slot(i, 1)], x[1])), __dmul_rn(q[slot(i, 2)], x[2])),
                     q[slot(i, 3)]);
  const double c = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x[0], r[0]), __dmul_rn(x[1], r[1])), __dmul_rn(x[2], r[2])), r[3]);
  return c > 0.0 ? c : 0.0;
}

// The minimiser of v^T q v (Gaussian elimination with partial pivoting) and its cost; a pivot at or below kPivotRel
// times the largest diagonal entry takes the best of pa, pb and their midpoint, ties in that order.
__device__ __forceinline__ double place(const double q[10], const double pa[3], const double pb[3], double x[3]) {
  double M[3][4];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) M[i][j] = q[slot(i, j)];
    M[i][3] = -q[slot(i, 3)];
  }
  const double tol = __dmul_rn(kPivotRel, fmax(fmax(fabs(M[0][0]), fabs(M[1][1])), fabs(M[2][2])));
  bool singular = false;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    double big = fabs(M[k][k]);  // the first row with the largest |M[i][k]| becomes row k
    int p = k;
#pragma unroll
    for (int i = k + 1; i < 3; ++i)
      if (fabs(M[i][k]) > big) {
        big = fabs(M[i][k]);
        p = i;
      }
    singular = singular || !(big > tol);
#pragma unroll
    for (int i = k + 1; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double t = M[k][j], u = M[i][j];
        M[k][j] = p == i ? u : t;
        M[i][j] = p == i ? t : u;
      }
#pragma unroll
    for (int i = k + 1; i < 3; ++i) {
      const double f = __ddiv_rn(M[i][k], M[k][k]);
#pragma unroll
      for (int j = k; j < 4; ++j) M[i][j] = __dsub_rn(M[i][j], __dmul_rn(f, M[k][j]));
    }
  }
  if (!singular) {
#pragma unroll
    for (int k = 2; k >= 0; --k) {
      double acc = M[k][3];
#pragma unroll
      for (int j = k + 1; j < 3; ++j) acc = __dsub_rn(acc, __dmul_rn(M[k][j], x[j]));
      x[k] = __ddiv_rn(acc, M[k][k]);
    }
    return quadric_cost(q, x);
  }
  double mid[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) mid[k] = __dmul_rn(__dadd_rn(pa[k], pb[k]), 0.5);
  double best = quadric_cost(q, pa);
  const double cb = quadric_cost(q, pb), cm = quadric_cost(q, mid);
  int pick = 0;
  if (cb < best) {
    best = cb;
    pick = 1;
  }
  if (cm < best) {
    best = cm;
    pick = 2;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) x[k] = pick == 0 ? pa[k] : pick == 1 ? pb[k] : mid[k];
  return best;
}

__device__ __forceinline__ void edge_quadric(const double* Q, int a, int b, double q[10]) {
#pragma unroll
  for (int t = 0; t < 10; ++t) q[t] = __dadd_rn(Q[10 * (size_t)a + t], Q[10 * (size_t)b + t]);
}

// ---- preparation and per-round structure ------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) prepare_kernel(const double* __restrict__ verts, const int64_t* __restrict__ faces, long long V,
                                                           long long F, int* __restrict__ fw, double* __restrict__ P, int* __restrict__ remap,
                                                           int* __restrict__ bad) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < 3 * F; i += stride) {
    const long long v = faces[i];
    if (v < 0 || v >= V) atomicOr(bad, 1);
    fw[i] = (int)v;
  }
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += stride) {
    #pragma unroll
    for (int k = 0; k < 3; ++k) P[3 * v + k] = verts[3 * v + k];
    remap[v] = (int)v;
  }
}

// half-edge h = 3f + k runs from corner k to corner (k + 1) % 3; corner h is vertex fw[h]
__global__ void __launch_bounds__(kThreads) half_edges_kernel(const int* __restrict__ fw, long long F, long long V, unsigned long long* __restrict__ ekeys,
                                                              int* __restrict__ evals, uint32_t* __restrict__ ikeys, int* __restrict__ ivals) {
  for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h < 3 * F; h += (long long)gridDim.x * blockDim.x) {
    const long long f = h / 3;
    const int k = (int)(h - 3 * f);
    const int a = fw[h], b = fw[3 * f + (k + 1) % 3];
    if (ekeys) {
      ekeys[h] = half_edge_key((unsigned long long)a, (unsigned long long)b, (unsigned long long)V);
      evals[h] = (int)h;
    }
    ikeys[h] = (uint32_t)a;
    ivals[h] = (int)h;
  }
}

__global__ void __launch_bounds__(kThreads) vstart_kernel(const uint32_t* __restrict__ ikeys, long long n, long long V, int* __restrict__ vstart) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v <= V; v += (long long)gridDim.x * blockDim.x) {
    long long lo = 0, hi = n;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (ikeys[mid] < (uint32_t)v) lo = mid + 1;
      else hi = mid;
    }
    vstart[v] = (int)lo;
  }
}

// edge runs of the sorted keys: slot i opens a run when its key differs from slot i - 1; the face count, up to 3
__device__ __forceinline__ int run_count(const unsigned long long* __restrict__ keys, long long n, long long i) {
  const unsigned long long key = keys[i];
  int c = 1;
  while (c < 3 && i + c < n && keys[i + c] == key) ++c;
  return c;
}

__device__ __forceinline__ bool run_start(const unsigned long long* __restrict__ keys, long long i) { return i == 0 || keys[i - 1] != keys[i]; }

__global__ void __launch_bounds__(kThreads) boundary_halfedges_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ evals,
                                                                      long long n, uint8_t* __restrict__ hb) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (run_start(keys, i) && run_count(keys, n, i) == 1) hb[evals[i]] = 1;
}

struct KMesh {
  const int* fw;        // [3F] faces
  const double* P;      // [3V] positions
  const int* vstart;    // [V+1]
  const int* corners;   // [3F] corners sorted by vertex, in face order
};

__global__ void __launch_bounds__(kThreads) quadric_kernel(KMesh m, const uint8_t* __restrict__ hb, long long V, double* __restrict__ Q) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    double s[10];
#pragma unroll
    for (int t = 0; t < 10; ++t) s[t] = 0.0;
    for (int j = m.vstart[v]; j < m.vstart[v + 1]; ++j) {
      const int h = m.corners[j], f = h / 3, k = h - 3 * f;
      double p[3][3], n[3];
      #pragma unroll
      for (int t = 0; t < 3; ++t) load3(m.P, m.fw[3 * f + t], p[t]);
      face_normal(p[0], p[1], p[2], n);
      double c[10];
#pragma unroll
      for (int t = 0; t < 10; ++t) c[t] = 0.0;
      add_plane(c, n, p[0], __dmul_rn(__dsqrt_rn(dot3(n, n)), 0.5));
      #pragma unroll
      for (int e = 0; e < 2; ++e) {  // the boundary half-edges leaving (k) and entering (k + 2) the corner
        const int he = e == 0 ? k : (k + 2) % 3;
        if (!hb[3 * f + he]) continue;
        double p0[3], p1[3], d[3], mm[3];
        load3(m.P, m.fw[3 * f + he], p0);
        load3(m.P, m.fw[3 * f + (he + 1) % 3], p1);
        sub3(p1, p0, d);
        cross3(d, n, mm);
        add_plane(c, mm, p0, __dmul_rn(kBoundaryWeight, dot3(d, d)));
      }
#pragma unroll
      for (int t = 0; t < 10; ++t) s[t] = __dadd_rn(s[t], c[t]);
    }
#pragma unroll
    for (int t = 0; t < 10; ++t) Q[10 * v + t] = s[t];
  }
}

__global__ void __launch_bounds__(kThreads) boundary_kernel(const unsigned long long* __restrict__ keys, long long n, long long V, int* __restrict__ onb) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (run_start(keys, i) && run_count(keys, n, i) == 1) {
      onb[keys[i] / (unsigned long long)V] = 1;
      onb[keys[i] % (unsigned long long)V] = 1;
    }
}

// ---- validity and cost ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool face_has(const int* fw, int f, int x) { return fw[3 * f] == x || fw[3 * f + 1] == x || fw[3 * f + 2] == x; }

// x shares a face with v
__device__ __forceinline__ bool in_star(const KMesh& m, int v, int x) {
  for (int j = m.vstart[v]; j < m.vstart[v + 1]; ++j)
    if (face_has(m.fw, m.corners[j] / 3, x)) return true;
  return false;
}

// |N(a) & N(b)|, counting up to limit + 1
__device__ __forceinline__ int common_neighbours(const KMesh& m, int a, int b, int limit) {
  int count = 0;
  const int j0 = m.vstart[a], j1 = m.vstart[a + 1];
  for (int j = j0; j < j1; ++j) {
    const int f = m.corners[j] / 3;
    #pragma unroll
    for (int t = 0; t < 3; ++t) {
      const int x = m.fw[3 * f + t];
      if (x == a || x == b) continue;
      bool seen = false;
      for (int u = 0; u < t && !seen; ++u) seen = m.fw[3 * f + u] == x;
      for (int jj = j0; jj < j && !seen; ++jj) seen = face_has(m.fw, m.corners[jj] / 3, x);
      if (seen || !in_star(m, b, x)) continue;
      if (++count > limit) return count;
    }
  }
  return count;
}

// no face around v that survives the collapse of (a, b) turns over or degenerates with a and b at x
__device__ __forceinline__ bool keeps_orientation(const KMesh& m, int v, int a, int b, const double x[3]) {
  for (int j = m.vstart[v]; j < m.vstart[v + 1]; ++j) {
    const int f = m.corners[j] / 3;
    const int* fv = m.fw + 3 * f;
    if (face_has(m.fw, f, a) && face_has(m.fw, f, b)) continue;
    double po[3][3], pn[3][3], no[3], nn[3];
    #pragma unroll
    for (int t = 0; t < 3; ++t) {
      load3(m.P, fv[t], po[t]);
      const bool moved = fv[t] == a || fv[t] == b;
      #pragma unroll
      for (int k = 0; k < 3; ++k) pn[t][k] = moved ? x[k] : po[t][k];
    }
    face_normal(po[0], po[1], po[2], no);
    face_normal(pn[0], pn[1], pn[2], nn);
    if (!(dot3(no, nn) > 0.0)) return false;
  }
  return true;
}

struct KRound {
  KMesh m;
  const double* Q;
  const unsigned long long* keys;  // [n] sorted half-edge keys
  const int* evals;                // [n] their half-edges
  const int* onb;                  // [V]
  long long n, V;
  unsigned long long* ckeys;       // [n] cost keys by slot
  int* cvals;                      // [n] slot
  int* num_valid;
};

__global__ void __launch_bounds__(kThreads) cost_kernel(KRound R) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < R.n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long out = kNoCost;
    R.cvals[i] = (int)i;
    if (run_start(R.keys, i)) {
      const int c = run_count(R.keys, R.n, i);
      const int a = (int)(R.keys[i] / (unsigned long long)R.V), b = (int)(R.keys[i] % (unsigned long long)R.V);
      bool ok = c <= 2 && a != b;
      if (ok && c == 2) {
        ok = !(R.onb[a] && R.onb[b]);
        if (ok) {
          const int h0 = R.evals[i], h1 = R.evals[i + 1];
          const int o1 = R.m.fw[3 * (h0 / 3) + (h0 % 3 + 2) % 3], o2 = R.m.fw[3 * (h1 / 3) + (h1 % 3 + 2) % 3];
          ok = o1 != o2 && !in_star(R.m, o1, o2);
        }
      }
      if (ok) ok = common_neighbours(R.m, a, b, c) == c;
      if (ok) {
        double q[10], pa[3], pb[3], x[3];
        edge_quadric(R.Q, a, b, q);
        load3(R.m.P, a, pa);
        load3(R.m.P, b, pb);
        const double cost = place(q, pa, pb, x);
        ok = keeps_orientation(R.m, a, a, b, x) && keeps_orientation(R.m, b, a, b, x);
        if (ok) {
          out = (unsigned long long)__double_as_longlong(cost);
          atomicAdd(R.num_valid, 1);
        }
      }
    }
    R.ckeys[i] = out;
  }
}

// ---- selection --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) fill_kernel(int* __restrict__ a, long long n, int value) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) a[i] = value;
}

// rank of each valid slot; m1[v] = least rank at v
__global__ void __launch_bounds__(kThreads) rank_kernel(const unsigned long long* __restrict__ sorted_cost, const int* __restrict__ sorted_slot,
                                                        const unsigned long long* __restrict__ keys, long long n, long long V, int* __restrict__ m1) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    if (sorted_cost[p] == kNoCost) continue;
    const unsigned long long key = keys[sorted_slot[p]];
    atomicMin(m1 + key / (unsigned long long)V, (int)p);
    atomicMin(m1 + key % (unsigned long long)V, (int)p);
  }
}

__global__ void __launch_bounds__(kThreads) m2_kernel(const unsigned long long* __restrict__ keys, long long n, long long V, const int* __restrict__ m1,
                                                      int* __restrict__ m2) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (!run_start(keys, i)) continue;
    const int a = (int)(keys[i] / (unsigned long long)V), b = (int)(keys[i] % (unsigned long long)V);
    atomicMin(m2 + a, m1[b]);
    atomicMin(m2 + b, m1[a]);
  }
}

// removed[p] = the face count of the edge of rank p when it is selected, else 0
__global__ void __launch_bounds__(kThreads) select_kernel(const unsigned long long* __restrict__ sorted_cost, const int* __restrict__ sorted_slot,
                                                          const unsigned long long* __restrict__ keys, long long n, long long V, const int* __restrict__ m2,
                                                          int* __restrict__ removed) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    int r = 0;
    if (sorted_cost[p] != kNoCost) {
      const long long i = sorted_slot[p];
      const unsigned long long key = keys[i];
      const int a = (int)(key / (unsigned long long)V), b = (int)(key % (unsigned long long)V);
      if (m2[a] == (int)p && m2[b] == (int)p) r = run_count(keys, n, i);
    }
    removed[p] = r;
  }
}

__global__ void __launch_bounds__(kThreads) collapse_kernel(const int* __restrict__ sorted_slot, const unsigned long long* __restrict__ keys, long long n,
                                                            long long V, const int* __restrict__ removed, const int* __restrict__ before, long long F,
                                                            long long target, double* P, double* Q, int* __restrict__ remap) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    if (removed[p] == 0 || F - before[p] <= target + 1) continue;
    const unsigned long long key = keys[sorted_slot[p]];
    const int a = (int)(key / (unsigned long long)V), b = (int)(key % (unsigned long long)V);
    double q[10], pa[3], pb[3], x[3];
    edge_quadric(Q, a, b, q);
    load3(P, a, pa);
    load3(P, b, pb);
    place(q, pa, pb, x);
    #pragma unroll
    for (int k = 0; k < 3; ++k) P[3 * (size_t)a + k] = x[k];
    #pragma unroll
    for (int t = 0; t < 10; ++t) Q[10 * (size_t)a + t] = q[t];
    remap[b] = a;
  }
}

__global__ void __launch_bounds__(kThreads) remap_kernel(int* __restrict__ fw, long long F, const int* __restrict__ remap, int* __restrict__ keep) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    const int a = remap[fw[3 * f]], b = remap[fw[3 * f + 1]], c = remap[fw[3 * f + 2]];
    fw[3 * f] = a;
    fw[3 * f + 1] = b;
    fw[3 * f + 2] = c;
    keep[f] = a != b && b != c && a != c;
  }
}

__global__ void __launch_bounds__(kThreads) compact_kernel(const int* __restrict__ fw, long long F, const int* __restrict__ keep, const int* __restrict__ at,
                                                           int* __restrict__ out, int* __restrict__ total) {
  for (long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x; f < F; f += (long long)gridDim.x * blockDim.x) {
    if (keep[f])
      #pragma unroll
      for (int k = 0; k < 3; ++k) out[3 * (size_t)at[f] + k] = fw[3 * f + k];
    if (f == F - 1) *total = at[f] + keep[f];
  }
}

// ---- output -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) used_kernel(const int* __restrict__ fw, long long n, int* __restrict__ used) {
  for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (long long)gridDim.x * blockDim.x) used[fw[h]] = 1;
}

__global__ void __launch_bounds__(kThreads) normals_kernel(KMesh m, long long V, const int* __restrict__ used, const int* __restrict__ at,
                                                           double* __restrict__ out_v, double* __restrict__ out_n, int* __restrict__ total) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    if (v == V - 1) *total = at[v] + used[v];
    if (!used[v]) continue;
    double s[3] = {0.0, 0.0, 0.0};
    for (int j = m.vstart[v]; j < m.vstart[v + 1]; ++j) {
      const int f = m.corners[j] / 3;
      double p[3][3], n[3];
      #pragma unroll
      for (int t = 0; t < 3; ++t) load3(m.P, m.fw[3 * f + t], p[t]);
      face_normal(p[0], p[1], p[2], n);
      #pragma unroll
      for (int k = 0; k < 3; ++k) s[k] = __dadd_rn(s[k], n[k]);
    }
    const double ln = __dsqrt_rn(dot3(s, s));
    const size_t o = 3 * (size_t)at[v];
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
      out_v[o + k] = m.P[3 * v + k];
      out_n[o + k] = ln > 0.0 ? __ddiv_rn(s[k], ln) : 0.0;
    }
  }
}

__global__ void __launch_bounds__(kThreads) out_faces_kernel(const int* __restrict__ fw, long long n, const int* __restrict__ at, int64_t* __restrict__ out) {
  for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h < n; h += (long long)gridDim.x * blockDim.x) out[h] = at[fw[h]];
}

// ---- host side --------------------------------------------------------------------------------------------------------
struct DScratch {
  double *P, *Q;                                 // [3V], [10V]
  int *remap, *m1, *m2, *onb, *used, *vat;      // [V]
  int* vstart;                                   // [V+1]
  int *fa, *fb;                                  // [3F] faces, ping-pong
  unsigned long long *ekeys_in, *ekeys;          // [3F]
  int *evals_in, *evals;                         // [3F]
  uint32_t *ikeys_in, *ikeys;                    // [3F]
  int *ivals_in, *ivals;                         // [3F]
  unsigned long long *ckeys_in, *ckeys;          // [3F]
  int *cvals_in, *cvals;                         // [3F]
  int *removed, *before;                         // [3F]
  uint8_t* hb;                                   // [3F]
  int *keep, *fat;                               // [F]
  int* counters;                                 // bad, valid edges, faces, vertices
  void* cub;
  size_t cub_bytes;
};

int decimate_cub_bytes(long long V, long long F, size_t* bytes) {
  size_t a = 0, b = 0, c = 0;
  const int nv = (int)std::max(V, 1LL), ne = (int)std::max(3 * F, 1LL);
  if (check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, a, (const int*)nullptr, (int*)nullptr, std::max(nv, ne)), "cub ExclusiveSum size query") ||
      check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const int*)nullptr,
                                                 (int*)nullptr, ne),
                 "cub SortPairs (edges) size query") ||
      check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, c, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr, (int*)nullptr, ne),
                 "cub SortPairs (corners) size query"))
    return FNR_ERR_CUDA;
  *bytes = std::max(a, std::max(b, c));
  return FNR_OK;
}

size_t dcarve(char* base, long long V, long long F, size_t cub_size, DScratch* s) {
  size_t off = 0;
  const size_t v = (size_t)std::max(V, 1LL), e = 3 * (size_t)std::max(F, 1LL), f = (size_t)std::max(F, 1LL);
  auto take = [&](size_t bytes) -> char* {
    char* p = base ? base + off : nullptr;
    off += (bytes + 255) / 256 * 256;
    return p;
  };
  s->P = (double*)take(24 * v);
  s->Q = (double*)take(80 * v);
  s->remap = (int*)take(4 * v);
  s->m1 = (int*)take(4 * v);
  s->m2 = (int*)take(4 * v);
  s->onb = (int*)take(4 * v);
  s->used = (int*)take(4 * v);
  s->vat = (int*)take(4 * v);
  s->vstart = (int*)take(4 * (v + 1));
  s->fa = (int*)take(4 * e);
  s->fb = (int*)take(4 * e);
  s->ekeys_in = (unsigned long long*)take(8 * e);
  s->ekeys = (unsigned long long*)take(8 * e);
  s->evals_in = (int*)take(4 * e);
  s->evals = (int*)take(4 * e);
  s->ikeys_in = (uint32_t*)take(4 * e);
  s->ikeys = (uint32_t*)take(4 * e);
  s->ivals_in = (int*)take(4 * e);
  s->ivals = (int*)take(4 * e);
  s->ckeys_in = (unsigned long long*)take(8 * e);
  s->ckeys = (unsigned long long*)take(8 * e);
  s->cvals_in = (int*)take(4 * e);
  s->cvals = (int*)take(4 * e);
  s->removed = (int*)take(4 * e);
  s->before = (int*)take(4 * e);
  s->hb = (uint8_t*)take(e);
  s->keep = (int*)take(4 * f);
  s->fat = (int*)take(4 * f);
  s->counters = (int*)take(16);
  s->cub = take(cub_size);
  s->cub_bytes = cub_size;
  return off;
}

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

// corners of the faces fw sorted by vertex, vstart; with ekeys the half-edges sorted by key as well
int sort_mesh(DScratch& s, const int* fw, long long F, long long V, bool edges, cudaStream_t st) {
  const long long n = 3 * F;
  FNR_LAUNCH(half_edges_kernel, n, fw, F, V, edges ? s.ekeys_in : nullptr, s.evals_in, s.ikeys_in, s.ivals_in);
  size_t tb = s.cub_bytes;
  if (edges) FNR_CUDA(sort_half_edges(s.cub, tb, s.ekeys_in, s.ekeys, s.evals_in, s.evals, n, V, st), "cub SortPairs (edges)");
  tb = s.cub_bytes;
  FNR_CUDA(cub::DeviceRadixSort::SortPairs(s.cub, tb, s.ikeys_in, s.ikeys, s.ivals_in, s.ivals, (int)n, 0, bits_for((unsigned long long)V + 1), st),
           "cub SortPairs (corners)");
  FNR_LAUNCH(vstart_kernel, V + 1, s.ikeys, n, V, s.vstart);
  return FNR_OK;
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_mesh_decimate_scratch_bytes(int64_t num_vertices, int64_t num_faces, size_t* bytes) {
  const char* what = "fnr_mesh_decimate_scratch_bytes";
  if (!bytes) {
    set_error("%s: NULL bytes", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_sizes(what, num_vertices, num_faces)) return rc;
  size_t cb = 0;
  if (int rc = decimate_cub_bytes(num_vertices, num_faces, &cb)) return rc;
  DScratch s;
  *bytes = dcarve(nullptr, num_vertices, num_faces, cb, &s);
  return FNR_OK;
}

int fnr_mesh_decimate(const double* vertices, const int64_t* faces, int64_t num_vertices, int64_t num_faces, int64_t target_num_faces, void* scratch,
                      size_t scratch_bytes, double* out_vertices, double* out_normals, int64_t* out_faces, int64_t* out_num_vertices,
                      int64_t* out_num_faces, int32_t* out_rounds, void* stream) {
  const char* what = "fnr_mesh_decimate";
  if ((num_vertices > 0 && (!vertices || !out_vertices || !out_normals)) || (num_faces > 0 && (!faces || !out_faces)) || !out_num_vertices ||
      !out_num_faces || !out_rounds) {
    set_error("%s: NULL arguments", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (int rc = check_sizes(what, num_vertices, num_faces)) return rc;
  if (target_num_faces < 1) {
    set_error("%s: target_num_faces must be >= 1, got %lld", what, (long long)target_num_faces);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  size_t cb = 0;
  if (int rc = decimate_cub_bytes(num_vertices, num_faces, &cb)) return rc;
  DScratch s;
  const size_t need = dcarve(nullptr, num_vertices, num_faces, cb, &s);
  if (!scratch || scratch_bytes < need) {
    set_error("%s: scratch too small: need %zu bytes, got %zu", what, need, scratch ? scratch_bytes : (size_t)0);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  dcarve(static_cast<char*>(scratch), num_vertices, num_faces, cb, &s);
  *out_num_vertices = 0;
  *out_num_faces = 0;
  *out_rounds = 0;
  if (num_faces == 0) return FNR_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long V = num_vertices, N = target_num_faces;
  long long F = num_faces;
  int host[4] = {0, 0, 0, 0};
  FNR_CUDA(cudaMemsetAsync(s.counters, 0, 4 * sizeof(int), st), "cudaMemsetAsync");
  FNR_LAUNCH(prepare_kernel, std::max(3 * F, V), vertices, faces, V, F, s.fa, s.P, s.remap, s.counters);
  FNR_CUDA(cudaMemcpyAsync(host, s.counters, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
  FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
  if (host[0]) {
    set_error("%s: a face index lies outside [0, %lld)", what, V);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  // quadrics of the input mesh
  if (int rc = sort_mesh(s, s.fa, F, V, true, st)) return rc;
  FNR_CUDA(cudaMemsetAsync(s.hb, 0, 3 * (size_t)F, st), "cudaMemsetAsync");
  FNR_LAUNCH(boundary_halfedges_kernel, 3 * F, s.ekeys, s.evals, 3 * F, s.hb);
  KMesh m{s.fa, s.P, s.vstart, s.ivals};
  FNR_LAUNCH(quadric_kernel, V, m, s.hb, V, s.Q);
  int rounds = 0;
  while (F > N + 1) {
    const long long n = 3 * F;
    if (rounds > 0)
      if (int rc = sort_mesh(s, s.fa, F, V, true, st)) return rc;
    FNR_CUDA(cudaMemsetAsync(s.onb, 0, sizeof(int) * (size_t)V, st), "cudaMemsetAsync");
    FNR_CUDA(cudaMemsetAsync(s.counters + 1, 0, 2 * sizeof(int), st), "cudaMemsetAsync");
    FNR_LAUNCH(boundary_kernel, n, s.ekeys, n, V, s.onb);
    m = KMesh{s.fa, s.P, s.vstart, s.ivals};
    KRound R{m, s.Q, s.ekeys, s.evals, s.onb, n, V, s.ckeys_in, s.cvals_in, s.counters + 1};
    FNR_LAUNCH(cost_kernel, n, R);
    size_t tb = s.cub_bytes;
    FNR_CUDA(cub::DeviceRadixSort::SortPairs(s.cub, tb, s.ckeys_in, s.ckeys, s.cvals_in, s.cvals, (int)n, 0, 63, st), "cub SortPairs (costs)");
    FNR_LAUNCH(fill_kernel, V, s.m1, V, INT_MAX);
    FNR_LAUNCH(rank_kernel, n, s.ckeys, s.cvals, s.ekeys, n, V, s.m1);
    FNR_CUDA(cudaMemcpyAsync(s.m2, s.m1, sizeof(int) * (size_t)V, cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync");
    FNR_LAUNCH(m2_kernel, n, s.ekeys, n, V, s.m1, s.m2);
    FNR_LAUNCH(select_kernel, n, s.ckeys, s.cvals, s.ekeys, n, V, s.m2, s.removed);
    tb = s.cub_bytes;
    FNR_CUDA(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.removed, s.before, (int)n, st), "cub ExclusiveSum (removed faces)");
    FNR_LAUNCH(collapse_kernel, n, s.cvals, s.ekeys, n, V, s.removed, s.before, F, N, s.P, s.Q, s.remap);
    FNR_LAUNCH(remap_kernel, F, s.fa, F, s.remap, s.keep);
    tb = s.cub_bytes;
    FNR_CUDA(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.keep, s.fat, (int)F, st), "cub ExclusiveSum (faces)");
    FNR_LAUNCH(compact_kernel, F, s.fa, F, s.keep, s.fat, s.fb, s.counters + 2);
    FNR_CUDA(cudaMemcpyAsync(host, s.counters, 4 * sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (host[1] == 0) break;  // no valid edge: nothing collapsed, the faces are as they were
    std::swap(s.fa, s.fb);
    F = host[2];
    ++rounds;
  }
  // drop unused vertices in input order, remap the faces, normals from the final faces
  if (int rc = sort_mesh(s, s.fa, F, V, false, st)) return rc;
  FNR_CUDA(cudaMemsetAsync(s.used, 0, sizeof(int) * (size_t)V, st), "cudaMemsetAsync");
  FNR_LAUNCH(used_kernel, 3 * F, s.fa, 3 * F, s.used);
  size_t tb = s.cub_bytes;
  FNR_CUDA(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.used, s.vat, (int)V, st), "cub ExclusiveSum (vertices)");
  m = KMesh{s.fa, s.P, s.vstart, s.ivals};
  FNR_LAUNCH(normals_kernel, V, m, V, s.used, s.vat, out_vertices, out_normals, s.counters + 3);
  FNR_LAUNCH(out_faces_kernel, 3 * F, s.fa, 3 * F, s.vat, out_faces);
  FNR_CUDA(cudaMemcpyAsync(host, s.counters, 4 * sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
  FNR_CUDA(cudaStreamSynchronize(st), "cudaStreamSynchronize");
  *out_num_vertices = host[3];
  *out_num_faces = F;
  *out_rounds = rounds;
  return FNR_OK;
}

}  // extern "C"
