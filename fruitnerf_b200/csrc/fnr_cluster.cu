// Fruit counting on the device: radius neighbour counts (radius-outlier removal and the DBSCAN core test), voxel
// down-sampling, DBSCAN labels and per-cluster sums -- stages 1-2 of the reference clustering
// (clustering/clustering_base.py:138-143, 183-259).  clustering.py's numpy / scikit-learn code is the oracle of every
// kernel here.
//
// Neighbour queries go through a uniform grid.  Cell keys (21 bits per axis) are radix-sorted with CUB, the points are
// gathered in key order (a stable sort: input order inside a cell) and a query walks the +-2 neighbourhood of its cell as
// 25 (x, y) columns, one binary search over the sorted unique keys per column.  For a radius r the cell side is
// h = (15/16) r / sqrt(3): every pair of points inside one cell is closer than r, and a pair within r is at most two cells
// apart on each axis (r / h = 1.85).  The 1/16 margin absorbs the rounding of the key arithmetic.
//
// The multi-radius call (fnr_radius_count_multi) answers R radii r_1..r_R on one grid whose side comes
// from the smallest radius, h = cell_side(r_min): the own cell is still within every radius, and a larger radius walks
// more rings.  The ring of radius r is ring(r) = floor(r/h + 1/16) + 1.  Derivation: the keys are floor(q) with q the
// computed (p - lo) / h; check_extent bounds |p| / h by 2^40 and the extent by 2^21 cells, so each q is within 2^-12 of
// its exact value and two points' q differ by at most r/h + 2^-11 < r/h + 1/16 when |dp| <= r on that axis (the fp64
// predicate d2 <= r*r admits |dp| only 2^-50 r beyond r).  Two integers floor(q1) <= floor(q2) then differ by
// D < r/h + 1/16 + 1, so D <= floor(r/h + 1/16) + 1.  For r = r_min this is the +-2 above (floor(1.85 + 0.06) + 1); the
// call accepts r_max / r_min <= 4, i.e. r_max / h <= 7.4 and at most 8 rings.
//
// Distances are fp64 with explicit round-to-nearest intrinsics in x, y, z order, d2 = (dx*dx + dy*dy) + dz*dz <= r*r:
// scikit-learn's KD-tree radius predicate bit for bit.  No host synchronisation; data-dependent sizes (cells, voxels,
// clusters) stay in device memory.
#include <cub/cub.cuh>
#include <math_constants.h>
#include <algorithm>
#include <climits>
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_grid.cuh"
#include "fnr_kernels.h"
#include "fnr_union_find.cuh"

namespace fnr {

namespace {

constexpr int kThreads = kGridThreads;
constexpr int kNone = 0x7fffffff;  // "no core point" / "no root": above every int32 point index
constexpr double kCellShrink = 15.0 / 16.0;
constexpr double kMaxCoordOverCell = 1099511627776.0;  // 2^40: beyond it a key's rounding error nears the 1/16 margin

// Calls f(cell, ring) for every occupied cell within +-reach cells of `key` on each axis, ring = Chebyshev distance in
// cells (0 = the cell itself).  f returns false to stop the walk.  The single-radius kernels walk +-2; the multi-radius
// count passes the ring of its largest radius (header comment).
template <class F>
__device__ __forceinline__ void for_each_near_cell(const Grid& g, int nc, uint64_t key, F&& f, int reach = 2) {
  const long long cx = (long long)(key >> (2 * kAxisBits)), cy = (long long)((key >> kAxisBits) & kAxisMask),
                  cz = (long long)(key & kAxisMask);
  for (int dx = -reach; dx <= reach; ++dx) {
    const long long x = cx + dx;
    if (x < 0 || x >= kAxisCells) continue;
    for (int dy = -reach; dy <= reach; ++dy) {
      const long long y = cy + dy;
      if (y < 0 || y >= kAxisCells) continue;
      const uint64_t hi = pack_key(x, y, cz + reach < kAxisCells ? cz + reach : kAxisCells - 1);
      const int dxy = max(abs(dx), abs(dy));
      for (int c = lower_bound(g.ukeys, nc, pack_key(x, y, cz > reach ? cz - reach : 0)); c < nc; ++c) {
        const uint64_t k = g.ukeys[c];
        if (k > hi) break;
        const int ring = max(dxy, (int)llabs((long long)(k & kAxisMask) - cz));
        if (!f(c, ring)) return;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) fill_kernel(int* __restrict__ a, int n, int v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// ---- radius neighbour count -----------------------------------------------------------------------------------------
// count = #{j : d2(i, j) <= r2} (i included), saturated at cap.  The own cell counts whole, without distance tests.
__global__ void __launch_bounds__(kThreads) radius_count_kernel(Grid g, double r2, int cap, int* __restrict__ counts,
                                                                int* __restrict__ core_sorted) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const int own = g.cell_of[j];
  int cnt = g.cstart[own + 1] - g.cstart[own];
  if (cnt < cap) {
    const double px = g.x[j], py = g.y[j], pz = g.z[j];
    for_each_near_cell(g, *g.ncells, g.keys[j], [&](int c, int ring) {
      if (ring == 0) return true;
      for (int k = g.cstart[c], e = g.cstart[c + 1]; k < e; ++k)
        if (dist2(px, py, pz, g.x[k], g.y[k], g.z[k]) <= r2 && ++cnt >= cap) return false;
      return true;
    });
  }
  cnt = min(cnt, cap);
  if (counts) counts[g.perm[j]] = cnt;
  if (core_sorted) core_sorted[j] = cnt >= cap;
}

// The radii of one multi-radius walk, passed by value (constant bank).  ring[k] = ring(r_k) of the header comment.
constexpr int kMaxRadii = 16;
struct Radii {
  double r2[kMaxRadii];
  int cap[kMaxRadii];
  int ring[kMaxRadii];
  int num;
  int reach;  // the largest ring
};

// radius_count_kernel for R <= kR radii on one grid: each pair's d2 is computed once and compared with every r_k^2 whose
// ring reaches its cell.  A point stops once every count has reached its cap.  counts: [R,n] rows in input order.
template <int kR>
__global__ void __launch_bounds__(kThreads) radius_count_multi_kernel(Grid g, Radii rs, int* __restrict__ counts) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const int own = g.cell_of[j];
  const int whole = g.cstart[own + 1] - g.cstart[own];
  int cnt[kR];
  int open = 0;  // counts still below their cap
#pragma unroll
  for (int k = 0; k < kR; ++k) {
    cnt[k] = whole;
    if (k < rs.num && whole < rs.cap[k]) ++open;
  }
  if (open) {
    const double px = g.x[j], py = g.y[j], pz = g.z[j];
    for_each_near_cell(g, *g.ncells, g.keys[j], [&](int c, int ring) {
      if (ring == 0) return true;
      for (int m = g.cstart[c], e = g.cstart[c + 1]; m < e; ++m) {
        const double d2 = dist2(px, py, pz, g.x[m], g.y[m], g.z[m]);
#pragma unroll
        for (int k = 0; k < kR; ++k)
          if (k < rs.num && ring <= rs.ring[k] && cnt[k] < rs.cap[k] && d2 <= rs.r2[k] && ++cnt[k] == rs.cap[k]) --open;
        if (!open) return false;
      }
      return true;
    }, rs.reach);
  }
  const size_t n = (size_t)g.n;
#pragma unroll
  for (int k = 0; k < kR; ++k) {
    if (k < rs.num) counts[k * n + g.perm[j]] = min(cnt[k], rs.cap[k]);
  }
}

// ---- DBSCAN ---------------------------------------------------------------------------------------------------------
// Union-find over input indices (fnr_union_find.cuh): the root of a component is its smallest core index.

__global__ void __launch_bounds__(kThreads) cell_min_core_kernel(Grid g, const int* __restrict__ core, int* __restrict__ cmin) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < g.n && core[j]) atomicMin(cmin + g.cell_of[j], g.perm[j]);
}

// The cores of one cell are mutually within eps: they start as one tree rooted at the cell's smallest core index.
__global__ void __launch_bounds__(kThreads) parent_init_kernel(Grid g, const int* __restrict__ core, const int* __restrict__ cmin,
                                                               int* __restrict__ parent) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const int i = g.perm[j];
  parent[i] = core[j] ? cmin[g.cell_of[j]] : i;
}

// Joins the core at sorted position j to the cores of every cell at Chebyshev distance `ring_sel` whose component still
// differs from its own: the first core pair within eps found in that cell hooks the two trees.
__global__ void __launch_bounds__(kThreads) link_kernel(Grid g, const int* __restrict__ core, const int* __restrict__ cmin, double e2,
                                                        int ring_sel, int* parent) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n || !core[j]) return;
  const int i = g.perm[j];
  const double px = g.x[j], py = g.y[j], pz = g.z[j];
  for_each_near_cell(g, *g.ncells, g.keys[j], [&](int c, int ring) {
    if (ring != ring_sel) return true;
    const int m = cmin[c];
    if (m == kNone || find_root(parent, i) == find_root(parent, m)) return true;
    for (int k = g.cstart[c], e = g.cstart[c + 1]; k < e; ++k) {
      if (core[k] && dist2(px, py, pz, g.x[k], g.y[k], g.z[k]) <= e2) {
        unite(parent, i, g.perm[k]);
        break;
      }
    }
    return true;
  });
}

// Points every node straight at its root; runs when no hooking is in flight, so the roots are fixed.  The walk only reads
// (a path-halving store from another thread could put a non-root ancestor back into a slot already set to its root) and
// each thread writes its own slot alone: when the kernel ends, parent[i] is the root of i for every i.
__global__ void __launch_bounds__(kThreads) flatten_kernel(int n, int* parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const volatile int* p = parent;
  int r = p[i];
  while (r != p[r]) r = p[r];  // a read may see an older or newer ancestor: both lead to the same root
  parent[i] = r;
}

__global__ void __launch_bounds__(kThreads) root_flag_kernel(Grid g, const int* __restrict__ core, const int* __restrict__ parent,
                                                             int* __restrict__ flag) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const int i = g.perm[j];
  flag[i] = core[j] && parent[i] == i;
}

// cid = exclusive scan of the root flags: clusters numbered in increasing order of their smallest core index, as
// scikit-learn's dbscan_inner discovers them.  A border point takes the cluster of the smallest root among the cores
// within eps (the first cluster whose expansion reaches it); everything else is noise (-1).
__global__ void __launch_bounds__(kThreads) label_kernel(Grid g, const int* __restrict__ core, const int* __restrict__ cmin,
                                                         const int* __restrict__ parent, const int* __restrict__ cid,
                                                         const int* __restrict__ flag, double e2, int32_t* __restrict__ labels,
                                                         int32_t* __restrict__ num_clusters) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const int i = g.perm[j];
  if (i == g.n - 1) *num_clusters = cid[i] + flag[i];
  if (core[j]) {
    labels[i] = cid[parent[i]];
    return;
  }
  const int own = g.cell_of[j];
  int best = cmin[own] == kNone ? kNone : parent[cmin[own]];
  const double px = g.x[j], py = g.y[j], pz = g.z[j];
  for_each_near_cell(g, *g.ncells, g.keys[j], [&](int c, int ring) {
    if (ring == 0 || cmin[c] == kNone) return true;
    const int root = parent[cmin[c]];
    if (root >= best) return true;  // every core of cell c is in this one component
    for (int k = g.cstart[c], e = g.cstart[c + 1]; k < e; ++k) {
      if (core[k] && dist2(px, py, pz, g.x[k], g.y[k], g.z[k]) <= e2) {
        best = root;
        break;
      }
    }
    return true;
  });
  labels[i] = best == kNone ? -1 : cid[best];
}

// ---- voxel down-sampling --------------------------------------------------------------------------------------------
// np.add.at(out, inv, points) / cnt: a sequential sum from 0.0 in input order (the stable sort kept it), then one division.
__global__ void __launch_bounds__(kThreads) voxel_mean_kernel(Grid g, double* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= *g.ncells) return;
  const int b = g.cstart[c], e = g.cstart[c + 1];
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (int k = b; k < e; ++k) {
    sx = __dadd_rn(sx, g.x[k]);
    sy = __dadd_rn(sy, g.y[k]);
    sz = __dadd_rn(sz, g.z[k]);
  }
  const double cnt = (double)(e - b);
  out[3 * (size_t)c] = __ddiv_rn(sx, cnt);
  out[3 * (size_t)c + 1] = __ddiv_rn(sy, cnt);
  out[3 * (size_t)c + 2] = __ddiv_rn(sz, cnt);
}

// ---- per-cluster sums -----------------------------------------------------------------------------------------------
// Labels outside [-1, K) are treated as noise.
__global__ void __launch_bounds__(kThreads) label_key_kernel(const int32_t* __restrict__ labels, int n, int K, uint32_t* __restrict__ keys,
                                                             int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = labels[i];
  keys[i] = (l >= 0 && l < K) ? (uint32_t)l + 1u : 0u;
  idx[i] = i;
}

// Points sorted by label (stable): cluster c owns sorted positions [start[c], end[c]).
__global__ void __launch_bounds__(kThreads) segment_bounds_kernel(int n, const uint32_t* __restrict__ skeys, int* __restrict__ start,
                                                                  int* __restrict__ end) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t k = skeys[j];
  if (k == 0) return;  // noise
  if (j == 0 || skeys[j - 1] != k) start[k - 1] = j;
  if (j == n - 1 || skeys[j + 1] != k) end[k - 1] = j + 1;
}

// One block per cluster, a fixed summation tree: the same input gives the same bits on every run.
__global__ void __launch_bounds__(kThreads) cluster_sums_kernel(const double* __restrict__ pts, const int* __restrict__ perm,
                                                                const int* __restrict__ start, const int* __restrict__ end, int K,
                                                                double* __restrict__ sums, int32_t* __restrict__ counts) {
  __shared__ double red[3][kThreads];
  const int t = threadIdx.x;
  for (int c = blockIdx.x; c < K; c += gridDim.x) {
    const int b = start[c], e = end[c];
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int k = b + t; k < e; k += kThreads) {
      const double* p = pts + 3 * (size_t)perm[k];
      s0 += p[0];
      s1 += p[1];
      s2 += p[2];
    }
    red[0][t] = s0;
    red[1][t] = s1;
    red[2][t] = s2;
    __syncthreads();
    for (int w = kThreads / 2; w > 0; w >>= 1) {
      if (t < w) {
        red[0][t] += red[0][t + w];
        red[1][t] += red[1][t + w];
        red[2][t] += red[2][t + w];
      }
      __syncthreads();
    }
    if (t == 0) {
      sums[3 * (size_t)c] = red[0][0];
      sums[3 * (size_t)c + 1] = red[1][0];
      sums[3 * (size_t)c + 2] = red[2][0];
      counts[c] = e - b;
    }
    __syncthreads();
  }
}

// ---- k nearest neighbours -------------------------------------------------------------------------------------------
// The point-cloud export's statistical outlier removal (k = 20) and normal estimation (k = 30): open3d's KD-tree kNN,
// exact.  A query walks Chebyshev rings of cells outward and keeps its k best (distance^2, input index) pairs, ordered
// by that pair, so ties go to the smaller index and every run gives the same list.
constexpr int kMaxK = 32;
constexpr int kKnnThreads = 128;
constexpr int kRingCap = 4;           // rings walked before a query moves to the exhaustive pass
constexpr double kRingMargin = 0.25;  // cells; key rounding moves a point by less than 2^-11 of a cell (check_extent)

// Calls f(cell) for every occupied cell at Chebyshev distance exactly `ring` from `key`: the side columns of the ring
// whole (one z range), the inner columns at their two z caps only (two one-cell ranges).  f has one call site, so the
// per-point work it inlines exists once.
template <class F>
__device__ __forceinline__ void for_each_cell_in_ring(const Grid& g, int nc, uint64_t key, int ring, F&& f) {
  const long long cx = (long long)(key >> (2 * kAxisBits)), cy = (long long)((key >> kAxisBits) & kAxisMask),
                  cz = (long long)(key & kAxisMask);
#pragma unroll 1
  for (int dx = -ring; dx <= ring; ++dx) {
    const long long x = cx + dx;
    if (x < 0 || x >= kAxisCells) continue;
#pragma unroll 1
    for (int dy = -ring; dy <= ring; ++dy) {
      const long long y = cy + dy;
      if (y < 0 || y >= kAxisCells) continue;
      const bool side = max(abs(dx), abs(dy)) == ring;
#pragma unroll 1
      for (int part = 0; part < (side ? 1 : 2); ++part) {
        long long zlo = part == 0 ? cz - ring : cz + ring;
        long long zhi = side ? cz + ring : zlo;
        if (zhi < 0 || zlo >= kAxisCells) continue;
        zlo = zlo < 0 ? 0 : zlo;
        zhi = zhi >= kAxisCells ? kAxisCells - 1 : zhi;
        const uint64_t hi = pack_key(x, y, zhi);
#pragma unroll 1
        for (int c = lower_bound(g.ukeys, nc, pack_key(x, y, zlo)); c < nc && g.ukeys[c] <= hi; ++c) f(c);
      }
    }
  }
}

__device__ __forceinline__ bool knn_less(double a, int ai, double b, int bi) { return a < b || (a == b && ai < bi); }

// The k best pairs in ascending order; entries k.. stay (+inf, kNone).  All indexing is static after unrolling, so the
// list lives in registers.
struct KnnList {
  double d[kMaxK];
  int i[kMaxK];
  double wd;  // the k-th entry, (+inf, kNone) until k pairs are in
  int wi;

  __device__ __forceinline__ void init() {
#pragma unroll
    for (int t = 0; t < kMaxK; ++t) {
      d[t] = CUDART_INF;
      i[t] = kNone;
    }
    wd = CUDART_INF;
    wi = kNone;
  }

  __device__ __forceinline__ void insert(int k, double nd, int ni) {
    if (!knn_less(nd, ni, wd, wi)) return;
#pragma unroll
    for (int t = kMaxK - 1; t > 0; --t) {  // descending: slot t reads the untouched slot t - 1
      if (t < k) {
        if (knn_less(nd, ni, d[t - 1], i[t - 1])) {
          d[t] = d[t - 1];
          i[t] = i[t - 1];
        } else if (knn_less(nd, ni, d[t], i[t])) {
          d[t] = nd;
          i[t] = ni;
        }
      }
    }
    if (knn_less(nd, ni, d[0], i[0])) {
      d[0] = nd;
      i[0] = ni;
    }
#pragma unroll
    for (int t = 0; t < kMaxK; ++t)
      if (t == k - 1) {
        wd = d[t];
        wi = i[t];
      }
  }
};

// Per-query result writers.  `i` is the input index of the query, L its k nearest neighbours (self included).
struct MeanDistanceOut {
  double* mean;
  __device__ __forceinline__ void finish(int i, const KnnList& L, int k) const {
    double s = 0.0;  // ascending, sequential: np.cumsum(d, axis=1)[:, -1]
#pragma unroll
    for (int t = 0; t < kMaxK; ++t)
      if (t < k) s = __dadd_rn(s, __dsqrt_rn(L.d[t]));
    mean[i] = __ddiv_rn(s, (double)k);
  }
};

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Direction of the null space of B - l*I for a symmetric 3x3 B (b = {b00, b01, b02, b11, b12, b22}): the largest cross
// product of two of its rows.  Returns that product's squared length (~0 when l is a double eigenvalue).
__device__ __forceinline__ double null_direction(const double* b, double l, double* v) {
  const double r[3][3] = {{b[0] - l, b[1], b[2]}, {b[1], b[3] - l, b[4]}, {b[2], b[4], b[5] - l}};
  double best = -1.0;
  for (int a = 0; a < 3; ++a) {
    double c[3];
    cross3(r[a], r[(a + 1) % 3], c);
    const double m = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
    if (m > best) {
      best = m;
      v[0] = c[0];
      v[1] = c[1];
      v[2] = c[2];
    }
  }
  return best;
}

// Unit eigenvector of the smallest eigenvalue of a symmetric 3x3 matrix (closed-form eigenvalues, then a null vector by
// cross products).  When the smallest eigenvalue is (numerically) double, every unit vector orthogonal to the largest
// eigenvalue's eigenvector is an answer, and one of them is returned.  The zero matrix and a multiple of the identity
// give (0, 0, 1).
__device__ __forceinline__ void smallest_eigenvector(const double* a, double* n) {
  n[0] = 0.0;
  n[1] = 0.0;
  n[2] = 1.0;
  double s = 0.0;
  for (int t = 0; t < 6; ++t) s = fmax(s, fabs(a[t]));
  if (!(s > 0.0)) return;
  double b[6];
  for (int t = 0; t < 6; ++t) b[t] = a[t] / s;
  const double q = (b[0] + b[3] + b[5]) / 3.0;
  const double p1 = b[1] * b[1] + b[2] * b[2] + b[4] * b[4];
  const double p2 = (b[0] - q) * (b[0] - q) + (b[3] - q) * (b[3] - q) + (b[5] - q) * (b[5] - q) + 2.0 * p1;
  if (!(p2 > 0.0)) return;
  const double p = sqrt(p2 / 6.0);
  const double c0 = (b[0] - q) / p, c1 = b[1] / p, c2 = b[2] / p, c3 = (b[3] - q) / p, c4 = b[4] / p, c5 = (b[5] - q) / p;
  const double det = c0 * (c3 * c5 - c4 * c4) - c1 * (c1 * c5 - c4 * c2) + c2 * (c1 * c4 - c3 * c2);
  const double r = fmin(1.0, fmax(-1.0, det / 2.0));
  const double phi = acos(r) / 3.0;
  const double l1 = q + 2.0 * p * cos(phi);                          // largest
  const double l3 = q + 2.0 * p * cos(phi + 2.0 * CUDART_PI / 3.0);  // smallest
  double v[3];
  if (!(null_direction(b, l3, v) > 1e-28)) {
    double u[3];
    if (!(null_direction(b, l1, u) > 1e-28)) return;
    if (fabs(u[0]) > fabs(u[1])) {
      v[0] = -u[2];
      v[1] = 0.0;
      v[2] = u[0];
    } else {
      v[0] = 0.0;
      v[1] = u[2];
      v[2] = -u[1];
    }
  }
  const double len = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (!(len > 0.0)) return;
  n[0] = v[0] / len;
  n[1] = v[1] / len;
  n[2] = v[2] / len;
}

// open3d EstimateNormals on the k nearest neighbours: fewer than 3 -> (0, 0, 1); else the smallest-eigenvalue
// eigenvector of their covariance (two passes: the mean, then the centred products).  With view directions, a normal
// whose fp32 dot product with its point's view direction is positive is flipped.
struct NormalsOut {
  const double* pts;  // input order
  const float* view;  // [n,3] or NULL
  double* normals;
  __device__ __forceinline__ void finish(int i, const KnnList& L, int k) const {
    double n[3] = {0.0, 0.0, 1.0};
    if (k >= 3) {
      double m[3] = {0.0, 0.0, 0.0};
#pragma unroll
      for (int t = 0; t < kMaxK; ++t)
        if (t < k) {
          const double* q = pts + 3 * (size_t)L.i[t];
          m[0] += q[0];
          m[1] += q[1];
          m[2] += q[2];
        }
      for (int a = 0; a < 3; ++a) m[a] /= (double)k;
      double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // c00 c01 c02 c11 c12 c22
#pragma unroll
      for (int t = 0; t < kMaxK; ++t)
        if (t < k) {
          const double* q = pts + 3 * (size_t)L.i[t];
          const double x = q[0] - m[0], y = q[1] - m[1], z = q[2] - m[2];
          c[0] += x * x;
          c[1] += x * y;
          c[2] += x * z;
          c[3] += y * y;
          c[4] += y * z;
          c[5] += z * z;
        }
      for (int a = 0; a < 6; ++a) c[a] /= (double)k;
      smallest_eigenvector(c, n);
    }
    if (view) {
      const float* v = view + 3 * (size_t)i;
      const float dot = __fadd_rn(__fadd_rn(__fmul_rn(v[0], __double2float_rn(n[0])), __fmul_rn(v[1], __double2float_rn(n[1]))),
                                  __fmul_rn(v[2], __double2float_rn(n[2])));
      if (dot > 0.0f) {
        n[0] = -n[0];
        n[1] = -n[1];
        n[2] = -n[2];
      }
    }
    double* o = normals + 3 * (size_t)i;
    o[0] = n[0];
    o[1] = n[1];
    o[2] = n[2];
  }
};

// One thread per query, in sorted order so a warp walks neighbouring cells.  After ring R every point not yet seen is
// at least (R - kRingMargin) * h away; the walk stops once the k-th distance is below that (or every point was seen).
// A query still open after kRingCap rings is queued for knn_exhaustive_kernel.
template <class Out>
__global__ void __launch_bounds__(kKnnThreads) knn_kernel(Grid g, int k, double h, Out out, int* __restrict__ open,
                                                          int* __restrict__ num_open) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const int nc = *g.ncells;
  const double px = g.x[j], py = g.y[j], pz = g.z[j];
  const uint64_t key = g.keys[j];
  KnnList L;
  L.init();
  int seen = 0;
#pragma unroll 1
  for (int ring = 0; ring <= kRingCap; ++ring) {
    for_each_cell_in_ring(g, nc, key, ring, [&](int c) {
      const int b = g.cstart[c], e = g.cstart[c + 1];
      seen += e - b;
#pragma unroll 1
      for (int m = b; m < e; ++m) L.insert(k, dist2(px, py, pz, g.x[m], g.y[m], g.z[m]), g.perm[m]);
    });
    const double bound = (ring - kRingMargin) * h;
    if (seen == g.n || (ring > 0 && L.wd < bound * bound * (1.0 - 1e-9))) {
      out.finish(g.perm[j], L, k);
      return;
    }
  }
  open[atomicAdd(num_open, 1)] = j;
}

// Exact pass for the queued queries, one block each: every thread keeps the best k of a strided share of all points,
// then k rounds of a block-wide minimum over the list heads merge them.
template <class Out>
__global__ void __launch_bounds__(kKnnThreads) knn_exhaustive_kernel(Grid g, int k, Out out, const int* __restrict__ open,
                                                                     const int* __restrict__ num_open) {
  __shared__ double sd[kKnnThreads];
  __shared__ int si[kKnnThreads], st[kKnnThreads];
  __shared__ double rd[kMaxK];
  __shared__ int ri[kMaxK];
  const int t = threadIdx.x;
  const int total = *num_open;
  for (int q = blockIdx.x; q < total; q += gridDim.x) {
    const int j = open[q];
    const double px = g.x[j], py = g.y[j], pz = g.z[j];
    KnnList L;
    L.init();
#pragma unroll 1
    for (int m = t; m < g.n; m += kKnnThreads) L.insert(k, dist2(px, py, pz, g.x[m], g.y[m], g.z[m]), g.perm[m]);
    int head = 0;
    for (int r = 0; r < k; ++r) {
      double hd = CUDART_INF;
      int hi = kNone;
#pragma unroll
      for (int u = 0; u < kMaxK; ++u)
        if (u == head) {
          hd = L.d[u];
          hi = L.i[u];
        }
      sd[t] = hd;
      si[t] = hi;
      st[t] = t;
      __syncthreads();
      for (int w = kKnnThreads / 2; w > 0; w >>= 1) {
        if (t < w && knn_less(sd[t + w], si[t + w], sd[t], si[t])) {
          sd[t] = sd[t + w];
          si[t] = si[t + w];
          st[t] = st[t + w];
        }
        __syncthreads();
      }
      if (t == st[0]) ++head;
      if (t == 0) {
        rd[r] = sd[0];
        ri[r] = si[0];
      }
      __syncthreads();
    }
    if (t == 0) {
#pragma unroll
      for (int u = 0; u < kMaxK; ++u)
        if (u < k) {
          L.d[u] = rd[u];
          L.i[u] = ri[u];
        }
      out.finish(g.perm[j], L, k);
    }
    __syncthreads();
  }
}

// ---- back-projection of rendered rays ---------------------------------------------------------------------------------
constexpr int kSelectThreads = 1024;

// point = origin + direction * depth (fp32, multiply then add, no FMA); keep accumulation > 0.5 and, with the box, every
// coordinate strictly inside it.  One block walks the batch in ray order and appends the kept rays at *count, so the
// rows come out in ray order; rows at or beyond `capacity` are counted but not written.
__global__ void __launch_bounds__(kSelectThreads) backproject_select_kernel(
    const float* __restrict__ origins, const float* __restrict__ directions, const float* __restrict__ depth,
    const float* __restrict__ rgb, const float* __restrict__ accumulation, int R, int use_box, float3 bmin, float3 bmax,
    int capacity, float* __restrict__ points, float* __restrict__ colors, float* __restrict__ view_dirs, int* __restrict__ count) {
  using Scan = cub::BlockScan<int, kSelectThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int base;
  if (threadIdx.x == 0) base = *count;
  __syncthreads();
  for (int r0 = 0; r0 < R; r0 += kSelectThreads) {
    const int r = r0 + threadIdx.x;
    float p[3];
    int keep = 0;
    if (r < R) {
      const float t = depth[r];
      for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(origins[3 * (size_t)r + a], __fmul_rn(directions[3 * (size_t)r + a], t));
      keep = accumulation[r] > 0.5f;
      if (use_box)
        keep = keep && p[0] > bmin.x && p[1] > bmin.y && p[2] > bmin.z && p[0] < bmax.x && p[1] < bmax.y && p[2] < bmax.z;
    }
    int pos, kept;
    Scan(tmp).ExclusiveSum(keep, pos, kept);
    if (keep && base + pos < capacity) {
      const size_t row = 3 * (size_t)(base + pos);
      for (int a = 0; a < 3; ++a) {
        points[row + a] = p[a];
        colors[row + a] = rgb[3 * (size_t)r + a];
        view_dirs[row + a] = directions[3 * (size_t)r + a];
      }
    }
    __syncthreads();  // every thread has read `base` and `tmp`
    if (threadIdx.x == 0) base += kept;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = base;
}

// ---- host side ------------------------------------------------------------------------------------------------------
// Caller-owned device scratch, carved in a fixed order (base == nullptr: sizes only): the grid's buffers, then DBSCAN's.
struct Scratch : GridBuffers {
  int* core;
  int* cmin;
  int* parent;
  int* cid;
};

int cub_bytes(int n, size_t* bytes) {
  size_t a = 0, b = 0, c = 0, d = 0;
  if (check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr, n),
                 "cub SortPairs (cell keys) size query") ||
      check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr, (int*)nullptr, n),
                 "cub SortPairs (labels) size query") ||
      check_cuda(cub::DeviceScan::InclusiveSum(nullptr, c, (const int*)nullptr, (int*)nullptr, n), "cub InclusiveSum size query") ||
      check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, d, (const int*)nullptr, (int*)nullptr, n), "cub ExclusiveSum size query"))
    return FNR_ERR_CUDA;
  *bytes = std::max(std::max(a, b), std::max(c, d));
  return FNR_OK;
}

size_t carve(char* base, int n, size_t cub_size, Scratch* s) {
  size_t off = 0;
  const size_t m = (size_t)(n > 0 ? n : 1);
  auto take = [&](size_t bytes) -> char* {
    char* p = base ? base + off : nullptr;
    off += (bytes + 255) / 256 * 256;
    return p;
  };
  s->keys_in = (uint64_t*)take(8 * m);
  s->keys = (uint64_t*)take(8 * m);
  s->idx_in = (int*)take(4 * m);
  s->perm = (int*)take(4 * m);
  s->x = (double*)take(8 * m);
  s->y = (double*)take(8 * m);
  s->z = (double*)take(8 * m);
  s->cell_of = (int*)take(4 * m);
  s->ukeys = (uint64_t*)take(8 * m);
  s->cstart = (int*)take(4 * (m + 1));
  s->ncells = (int*)take(4);
  s->core = (int*)take(4 * m);
  s->cmin = (int*)take(4 * m);
  s->parent = (int*)take(4 * m);
  s->flag = (int*)take(4 * m);
  s->cid = (int*)take(4 * m);
  s->cub = take(cub_size);
  s->cub_bytes = cub_size;
  return off;
}

int check_points(const char* what, const double* points, int64_t n, const double* lo, const double* hi) {
  if (n < 0 || n > 2147483647LL) {
    set_error("%s: point count %lld outside [0, 2^31 - 1]", what, (long long)n);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (n > 0 && (!points || !lo || !hi)) {
    set_error("%s: NULL points or bounds", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  for (int a = 0; n > 0 && a < 3; ++a) {
    if (!std::isfinite(lo[a]) || !std::isfinite(hi[a]) || hi[a] < lo[a]) {
      set_error("%s: invalid bounds on axis %d: [%g, %g]", what, a, lo[a], hi[a]);
      return FNR_ERR_INVALID_ARGUMENT;
    }
  }
  return FNR_OK;
}

int bind_scratch(const char* what, int n, void* scratch, size_t scratch_bytes, Scratch* s) {
  size_t cb = 0;
  if (int rc = cub_bytes(n, &cb)) return rc;
  const size_t need = carve(nullptr, n, cb, s);
  if (!scratch || scratch_bytes < need) {
    set_error("%s: scratch too small: need %zu bytes, got %zu", what, need, scratch ? scratch_bytes : (size_t)0);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  carve(static_cast<char*>(scratch), n, cb, s);
  return FNR_OK;
}

// Refuses extents that need more than 2^21 cells of side h on an axis (the key width).  `what_len` names the length
// the cell side derives from (the radius, eps or the voxel size).
int check_extent(const char* what, const char* what_len, double len, double h, const double* lo, const double* hi) {
  if (!(h > 0.0) || !std::isfinite(h)) {
    set_error("%s: %s must be positive and finite, got %g", what, what_len, len);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  for (int a = 0; a < 3; ++a) {
    const double cells = std::floor((hi[a] - lo[a]) / h);
    if (cells > (double)(kAxisCells - 1)) {
      set_error("%s: %s %g over an extent of %g on axis %d needs %.0f grid cells; at most 2^21 per axis are supported", what, what_len,
                len, hi[a] - lo[a], a, cells + 1);
      return FNR_ERR_UNSUPPORTED;
    }
    if (std::fmax(std::fabs(lo[a]), std::fabs(hi[a])) / h > kMaxCoordOverCell) {
      set_error("%s: %s %g is too small for coordinates of magnitude %g on axis %d (more than 2^40 cells from the origin)", what,
                what_len, len, std::fmax(std::fabs(lo[a]), std::fabs(hi[a])), a);
      return FNR_ERR_UNSUPPORTED;
    }
  }
  return FNR_OK;
}

double cell_side(double r) { return kCellShrink * r / std::sqrt(3.0); }

// ---- multi-radius count ---------------------------------------------------------------------------------------------
constexpr double kMaxRadiusRatio = 4.0;  // r_max / r_min: at most 8 rings (header comment)

// Checks R radii (`what_r`: their name) and caps and fills the walk parameters for the grid of side
// h = cell_side(r_min); *r_min receives r_min.
int make_radii(const char* what, const char* what_r, const double* radii, const int32_t* caps, int32_t num, Radii* rs, double* r_min) {
  if (num < 1 || !radii || !caps) {
    set_error("%s: %d radii with %s radii / caps; at least one, with non-NULL host arrays, is needed", what, num,
              radii && caps ? "" : "NULL ");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num > kMaxRadii) {
    set_error("%s: %d radii; at most %d are supported", what, num, kMaxRadii);
    return FNR_ERR_UNSUPPORTED;
  }
  double lo = radii[0], hi = radii[0];
  for (int k = 0; k < num; ++k) {
    if (!(radii[k] > 0.0) || !std::isfinite(radii[k]) || caps[k] < 1) {
      set_error("%s: %s %d is %g with cap %d; %s must be positive and finite and caps >= 1", what, what_r, k, radii[k], caps[k], what_r);
      return FNR_ERR_INVALID_ARGUMENT;
    }
    lo = std::fmin(lo, radii[k]);
    hi = std::fmax(hi, radii[k]);
  }
  if (hi > kMaxRadiusRatio * lo) {
    set_error("%s: largest %s %g is %g times the smallest %g; at most %g is supported", what, what_r, hi, hi / lo, lo, kMaxRadiusRatio);
    return FNR_ERR_UNSUPPORTED;
  }
  const double h = cell_side(lo);
  *rs = Radii{};
  rs->num = num;
  for (int k = 0; k < num; ++k) {
    rs->r2[k] = radii[k] * radii[k];
    rs->cap[k] = caps[k];
    rs->ring[k] = (int)std::floor(radii[k] / h + 1.0 / 16.0) + 1;
    rs->reach = std::max(rs->reach, rs->ring[k]);
  }
  *r_min = lo;
  return FNR_OK;
}

int launch_radius_count_multi(const Grid& g, int n, const Radii& rs, int* counts, cudaStream_t st) {
  const int nb = grid_for(n, kThreads, INT_MAX);
  if (rs.num <= 1) radius_count_multi_kernel<1><<<nb, kThreads, 0, st>>>(g, rs, counts);
  else if (rs.num <= 2) radius_count_multi_kernel<2><<<nb, kThreads, 0, st>>>(g, rs, counts);
  else if (rs.num <= 4) radius_count_multi_kernel<4><<<nb, kThreads, 0, st>>>(g, rs, counts);
  else if (rs.num <= 8) radius_count_multi_kernel<8><<<nb, kThreads, 0, st>>>(g, rs, counts);
  else radius_count_multi_kernel<kMaxRadii><<<nb, kThreads, 0, st>>>(g, rs, counts);
  return check_launch("radius_count_multi_kernel");
}

// Cell side of the kNN grid, from n, k and the bounds alone (no device read-back): the side at which k points would
// share a cell if the n points filled the bounding box evenly, taken over the box itself and over its largest face and
// longest edge (the largest of the three, so flat and thin clouds get cells sized for their own dimension).  It is then
// raised to the smallest side the keys allow: at most 2^21 - 1 cells per axis and 2^39 cells from the origin.  The
// rule sets the cost of a query, never its result.
double knn_cell_side(int n, int k, const double* lo, const double* hi) {
  double e[3] = {hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
  std::sort(e, e + 3, [](double a, double b) { return a > b; });
  double h = 0.0, prod = 1.0;
  for (int d = 1; d <= 3; ++d) {
    prod *= e[d - 1];
    if (prod > 0.0) h = std::fmax(h, std::pow(prod * k / n, 1.0 / d));
  }
  for (int a = 0; a < 3; ++a) {
    h = std::fmax(h, (hi[a] - lo[a]) / (double)(kAxisCells - 2));
    h = std::fmax(h, std::fmax(std::fabs(lo[a]), std::fabs(hi[a])) / (kMaxCoordOverCell / 2.0));
  }
  return h > 0.0 && std::isfinite(h) ? h : 1.0;  // all points identical: one cell
}

template <class Out>
int run_knn(const char* what, const double* points, int64_t num_points, const double* lo, const double* hi, int32_t k, bool out_ok,
            const Out& out, void* scratch, size_t scratch_bytes, void* stream) {
  if (int rc = check_points(what, points, num_points, lo, hi)) return rc;
  if (k < 1 || (num_points > 0 && !out_ok)) {
    set_error("%s: k must be >= 1 and the output non-NULL (k %d)", what, k);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (k > kMaxK) {
    set_error("%s: k = %d neighbours; at most %d are supported", what, k, kMaxK);
    return FNR_ERR_UNSUPPORTED;
  }
  const int n = (int)num_points;
  if (n == 0) return FNR_OK;
  const int kk = std::min(k, n);
  const double h = knn_cell_side(n, kk, lo, hi);
  if (int rc = check_extent(what, "kNN cell side", h, h, lo, hi)) return rc;
  Scratch s;
  if (int rc = bind_scratch(what, n, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Grid g;
  if (int rc = build_grid(points, n, lo, h, s, st, &g)) return rc;
  // the DBSCAN regions are free here: `core` holds the queue of open queries, `cmin[0]` its length
  if (int rc = check_cuda(cudaMemsetAsync(s.cmin, 0, sizeof(int), st), "kNN queue reset")) return rc;
  knn_kernel<Out><<<(n + kKnnThreads - 1) / kKnnThreads, kKnnThreads, 0, st>>>(g, kk, h, out, s.core, s.cmin);
  if (int rc = check_launch("knn_kernel")) return rc;
  knn_exhaustive_kernel<Out><<<std::min(n, 4 * sm_count()), kKnnThreads, 0, st>>>(g, kk, out, s.core, s.cmin);
  return check_launch("knn_exhaustive_kernel");
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_cluster_scratch_bytes(int64_t num_points, size_t* bytes) {
  if (!bytes || num_points < 0 || num_points > 2147483647LL) {
    set_error("invalid arguments to fnr_cluster_scratch_bytes (n = %lld)", (long long)num_points);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  size_t cb = 0;
  if (int rc = cub_bytes((int)num_points, &cb)) return rc;
  Scratch s;
  *bytes = carve(nullptr, (int)num_points, cb, &s);
  return FNR_OK;
}

int fnr_radius_count(const double* points, int64_t num_points, const double* lo, const double* hi, double radius, int32_t cap,
                     int32_t* counts, void* scratch, size_t scratch_bytes, void* stream) {
  const char* what = "fnr_radius_count";
  if (int rc = check_points(what, points, num_points, lo, hi)) return rc;
  if (cap < 1 || (num_points > 0 && !counts)) {
    set_error("%s: cap must be >= 1 and counts non-NULL (cap %d)", what, cap);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const int n = (int)num_points;
  if (n == 0) return FNR_OK;
  const double h = cell_side(radius);
  if (int rc = check_extent(what, "radius", radius, h, lo, hi)) return rc;
  Scratch s;
  if (int rc = bind_scratch(what, n, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Grid g;
  if (int rc = build_grid(points, n, lo, h, s, st, &g)) return rc;
  radius_count_kernel<<<grid_for(n, kThreads, INT_MAX), kThreads, 0, st>>>(g, radius * radius, cap, counts, nullptr);
  return check_launch("radius_count_kernel");
}

int fnr_voxel_down_sample(const double* points, int64_t num_points, const double* lo, const double* hi, double voxel, double* out,
                          int32_t* num_out, void* scratch, size_t scratch_bytes, void* stream) {
  const char* what = "fnr_voxel_down_sample";
  if (int rc = check_points(what, points, num_points, lo, hi)) return rc;
  if (!num_out || (num_points > 0 && !out)) {
    set_error("%s: NULL output", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n = (int)num_points;
  if (n == 0) return check_cuda(cudaMemsetAsync(num_out, 0, sizeof(int32_t), st), "fnr_voxel_down_sample (empty)");
  if (int rc = check_extent(what, "voxel size", voxel, voxel, lo, hi)) return rc;
  Scratch s;
  if (int rc = bind_scratch(what, n, scratch, scratch_bytes, &s)) return rc;
  Grid g;
  if (int rc = build_grid(points, n, lo, voxel, s, st, &g)) return rc;
  voxel_mean_kernel<<<grid_for(n, kThreads, INT_MAX), kThreads, 0, st>>>(g, out);
  if (int rc = check_launch("voxel_mean_kernel")) return rc;
  return check_cuda(cudaMemcpyAsync(num_out, s.ncells, sizeof(int32_t), cudaMemcpyDeviceToDevice, st), "fnr_voxel_down_sample (count)");
}

int fnr_dbscan(const double* points, int64_t num_points, const double* lo, const double* hi, double eps, int32_t min_samples,
               int32_t* labels, int32_t* num_clusters, void* scratch, size_t scratch_bytes, void* stream) {
  const char* what = "fnr_dbscan";
  if (int rc = check_points(what, points, num_points, lo, hi)) return rc;
  if (min_samples < 1 || !num_clusters || (num_points > 0 && !labels)) {
    set_error("%s: min_samples must be >= 1 and the outputs non-NULL (min_samples %d)", what, min_samples);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n = (int)num_points;
  if (n == 0) return check_cuda(cudaMemsetAsync(num_clusters, 0, sizeof(int32_t), st), "fnr_dbscan (empty)");
  const double h = cell_side(eps);
  if (int rc = check_extent(what, "eps", eps, h, lo, hi)) return rc;
  Scratch s;
  if (int rc = bind_scratch(what, n, scratch, scratch_bytes, &s)) return rc;
  Grid g;
  if (int rc = build_grid(points, n, lo, h, s, st, &g)) return rc;
  const double e2 = eps * eps;
  const int nb = grid_for(n, kThreads, INT_MAX);
  radius_count_kernel<<<nb, kThreads, 0, st>>>(g, e2, min_samples, nullptr, s.core);
  if (int rc = check_launch("radius_count_kernel")) return rc;
  fill_kernel<<<nb, kThreads, 0, st>>>(s.cmin, n, kNone);
  if (int rc = check_launch("fill_kernel")) return rc;
  cell_min_core_kernel<<<nb, kThreads, 0, st>>>(g, s.core, s.cmin);
  if (int rc = check_launch("cell_min_core_kernel")) return rc;
  parent_init_kernel<<<nb, kThreads, 0, st>>>(g, s.core, s.cmin, s.parent);
  if (int rc = check_launch("parent_init_kernel")) return rc;
  // face / edge / corner neighbours first (nearly every such cell pair links), then the cells two apart, most of which
  // the first pass has already put in the same component
  for (int ring = 1; ring <= 2; ++ring) {
    link_kernel<<<nb, kThreads, 0, st>>>(g, s.core, s.cmin, e2, ring, s.parent);
    if (int rc = check_launch("link_kernel")) return rc;
    flatten_kernel<<<nb, kThreads, 0, st>>>(n, s.parent);
    if (int rc = check_launch("flatten_kernel")) return rc;
  }
  root_flag_kernel<<<nb, kThreads, 0, st>>>(g, s.core, s.parent, s.flag);
  if (int rc = check_launch("root_flag_kernel")) return rc;
  size_t tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceScan::ExclusiveSum(s.cub, tb, s.flag, s.cid, n, st), "cub ExclusiveSum (cluster ids)")) return rc;
  label_kernel<<<nb, kThreads, 0, st>>>(g, s.core, s.cmin, s.parent, s.cid, s.flag, e2, labels, num_clusters);
  return check_launch("label_kernel");
}

int fnr_radius_count_multi(const double* points, int64_t num_points, const double* lo, const double* hi, const double* radii,
                           const int32_t* caps, int32_t num_radii, int32_t* counts, void* scratch, size_t scratch_bytes, void* stream) {
  const char* what = "fnr_radius_count_multi";
  if (int rc = check_points(what, points, num_points, lo, hi)) return rc;
  Radii rs;
  double r_min = 0.0;
  if (int rc = make_radii(what, "radius", radii, caps, num_radii, &rs, &r_min)) return rc;
  if (num_points > 0 && !counts) {
    set_error("%s: NULL counts", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const int n = (int)num_points;
  if (n == 0) return FNR_OK;
  const double h = cell_side(r_min);
  if (int rc = check_extent(what, "smallest radius", r_min, h, lo, hi)) return rc;
  Scratch s;
  if (int rc = bind_scratch(what, n, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Grid g;
  if (int rc = build_grid(points, n, lo, h, s, st, &g)) return rc;
  return launch_radius_count_multi(g, n, rs, counts, st);
}

int fnr_cluster_sums(const double* points, const int32_t* labels, int64_t num_points, int32_t num_clusters, double* sums,
                     int32_t* counts, void* scratch, size_t scratch_bytes, void* stream) {
  const char* what = "fnr_cluster_sums";
  if (num_points < 0 || num_points > 2147483647LL || num_clusters < 0 || num_clusters > num_points ||
      (num_points > 0 && (!points || !labels)) || (num_clusters > 0 && (!sums || !counts))) {
    set_error("%s: invalid arguments (n %lld, clusters %d)", what, (long long)num_points, num_clusters);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const int n = (int)num_points, K = num_clusters;
  if (K == 0) return FNR_OK;
  Scratch s;
  if (int rc = bind_scratch(what, n, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // sort key = label + 1 (noise first), stable: every cluster's points stay in input order
  uint32_t* kin = reinterpret_cast<uint32_t*>(s.keys_in);
  uint32_t* kout = reinterpret_cast<uint32_t*>(s.keys);
  const int nb = grid_for(n, kThreads, INT_MAX);
  label_key_kernel<<<nb, kThreads, 0, st>>>(labels, n, K, kin, s.idx_in);
  if (int rc = check_launch("label_key_kernel")) return rc;
  int bits = 1;
  while (bits < 32 && (1ull << bits) <= (unsigned long long)K) ++bits;  // keys are 0..K
  size_t tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceRadixSort::SortPairs(s.cub, tb, kin, kout, s.idx_in, s.perm, n, 0, bits, st), "cub SortPairs (labels)"))
    return rc;
  for (int* b : {s.cstart, s.cell_of}) {  // an id no point carries sums to zero
    fill_kernel<<<grid_for(K, kThreads, INT_MAX), kThreads, 0, st>>>(b, K, 0);
    if (int rc = check_launch("fill_kernel")) return rc;
  }
  segment_bounds_kernel<<<nb, kThreads, 0, st>>>(n, kout, s.cstart, s.cell_of);
  if (int rc = check_launch("segment_bounds_kernel")) return rc;
  cluster_sums_kernel<<<std::min(K, 8 * sm_count()), kThreads, 0, st>>>(points, s.perm, s.cstart, s.cell_of, K, sums, counts);
  return check_launch("cluster_sums_kernel");
}

int fnr_knn_mean_distance(const double* points, int64_t num_points, const double* lo, const double* hi, int32_t k, double* mean_dist,
                          void* scratch, size_t scratch_bytes, void* stream) {
  return run_knn("fnr_knn_mean_distance", points, num_points, lo, hi, k, mean_dist != nullptr, MeanDistanceOut{mean_dist}, scratch,
                 scratch_bytes, stream);
}

int fnr_estimate_normals(const double* points, int64_t num_points, const double* lo, const double* hi, int32_t k, const float* view_dirs,
                         double* normals, void* scratch, size_t scratch_bytes, void* stream) {
  return run_knn("fnr_estimate_normals", points, num_points, lo, hi, k, normals != nullptr, NormalsOut{points, view_dirs, normals},
                 scratch, scratch_bytes, stream);
}

int fnr_backproject_select(const float* origins, const float* directions, const float* depth, const float* rgb, const float* accumulation,
                           int32_t num_rays, int32_t use_bounding_box, const float* box_min, const float* box_max, int32_t capacity,
                           float* points, float* colors, float* view_dirs, int32_t* count, void* stream) {
  const char* what = "fnr_backproject_select";
  if (num_rays < 0 || capacity < 0 || !count || (use_bounding_box && (!box_min || !box_max)) ||
      (num_rays > 0 && (!origins || !directions || !depth || !rgb || !accumulation)) ||
      (capacity > 0 && (!points || !colors || !view_dirs))) {
    set_error("%s: invalid arguments (rays %d, capacity %d)", what, num_rays, capacity);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_rays == 0) return FNR_OK;
  const float3 bmin = use_bounding_box ? make_float3(box_min[0], box_min[1], box_min[2]) : make_float3(0.f, 0.f, 0.f);
  const float3 bmax = use_bounding_box ? make_float3(box_max[0], box_max[1], box_max[2]) : make_float3(0.f, 0.f, 0.f);
  backproject_select_kernel<<<1, kSelectThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      origins, directions, depth, rgb, accumulation, num_rays, use_bounding_box ? 1 : 0, bmin, bmax, capacity, points, colors, view_dirs, count);
  return check_launch("backproject_select_kernel");
}

}  // extern "C"
