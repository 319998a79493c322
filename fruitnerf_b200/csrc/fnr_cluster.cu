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
// Distances are fp64 with explicit round-to-nearest intrinsics in x, y, z order, d2 = (dx*dx + dy*dy) + dz*dz <= r*r:
// scikit-learn's KD-tree radius predicate bit for bit.  No host synchronisation; data-dependent sizes (cells, voxels,
// clusters) stay in device memory.
#include <cub/cub.cuh>
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kAxisBits = 21;
constexpr long long kAxisCells = 1LL << kAxisBits;
constexpr uint64_t kAxisMask = (uint64_t)kAxisCells - 1;
constexpr int kNone = 0x7fffffff;  // "no core point" / "no root": above every int32 point index
constexpr double kCellShrink = 15.0 / 16.0;
constexpr double kMaxCoordOverCell = 1099511627776.0;  // 2^40: beyond it a key's rounding error nears the 1/16 margin

__device__ __forceinline__ uint64_t pack_key(long long x, long long y, long long z) {
  return ((uint64_t)x << (2 * kAxisBits)) | ((uint64_t)y << kAxisBits) | (uint64_t)z;
}

__device__ __forceinline__ double dist2(double ax, double ay, double az, double bx, double by, double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// floor((p - origin) / h), clamped into the key range: the per-axis voxel key of clustering.voxel_down_sample
__device__ __forceinline__ long long axis_cell(double p, double origin, double h) {
  const double c = floor(__ddiv_rn(__dsub_rn(p, origin), h));
  return c < 0.0 ? 0 : (c > (double)(kAxisCells - 1) ? kAxisCells - 1 : (long long)c);
}

// The grid as the query kernels see it: sorted positions j = 0..n-1, cells c = 0..*ncells-1.
struct Grid {
  int n;
  const uint64_t* keys;   // [n] cell key of sorted position j
  const int* perm;        // [n] input index of sorted position j
  const double* x;        // [n] sorted coordinates
  const double* y;
  const double* z;
  const int* cell_of;     // [n] cell of sorted position j
  const uint64_t* ukeys;  // [ncells] sorted unique keys
  const int* cstart;      // [ncells + 1] first sorted position of each cell
  const int* ncells;      // device scalar
};

__device__ __forceinline__ int lower_bound(const uint64_t* __restrict__ a, int n, uint64_t k) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Calls f(cell, ring) for every occupied cell within +-2 cells of `key` on each axis, ring = Chebyshev distance in cells
// (0 = the cell itself).  f returns false to stop the walk.
template <class F>
__device__ __forceinline__ void for_each_near_cell(const Grid& g, int nc, uint64_t key, F&& f) {
  const long long cx = (long long)(key >> (2 * kAxisBits)), cy = (long long)((key >> kAxisBits) & kAxisMask),
                  cz = (long long)(key & kAxisMask);
  for (int dx = -2; dx <= 2; ++dx) {
    const long long x = cx + dx;
    if (x < 0 || x >= kAxisCells) continue;
    for (int dy = -2; dy <= 2; ++dy) {
      const long long y = cy + dy;
      if (y < 0 || y >= kAxisCells) continue;
      const uint64_t hi = pack_key(x, y, cz + 2 < kAxisCells ? cz + 2 : kAxisCells - 1);
      const int dxy = max(abs(dx), abs(dy));
      for (int c = lower_bound(g.ukeys, nc, pack_key(x, y, cz > 2 ? cz - 2 : 0)); c < nc; ++c) {
        const uint64_t k = g.ukeys[c];
        if (k > hi) break;
        const int ring = max(dxy, (int)llabs((long long)(k & kAxisMask) - cz));
        if (!f(c, ring)) return;
      }
    }
  }
}

// ---- grid construction ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) cell_key_kernel(const double* __restrict__ pts, int n, double ox, double oy, double oz,
                                                            double h, uint64_t* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* p = pts + 3 * (size_t)i;
  keys[i] = pack_key(axis_cell(p[0], ox, h), axis_cell(p[1], oy, h), axis_cell(p[2], oz, h));
  idx[i] = i;
}

// sorted coordinates + "first of its cell" flags (inclusive-scanned into cell_of afterwards)
__global__ void __launch_bounds__(kThreads) gather_kernel(const double* __restrict__ pts, int n, const uint64_t* __restrict__ keys,
                                                          const int* __restrict__ perm, double* __restrict__ x, double* __restrict__ y,
                                                          double* __restrict__ z, int* __restrict__ first) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double* p = pts + 3 * (size_t)perm[j];
  x[j] = p[0];
  y[j] = p[1];
  z[j] = p[2];
  first[j] = j == 0 || keys[j] != keys[j - 1];
}

// cell_of holds the inclusive scan of the flags on entry and the 0-based cell of each sorted position on exit
__global__ void __launch_bounds__(kThreads) cells_kernel(int n, const uint64_t* __restrict__ keys, int* __restrict__ cell_of,
                                                         uint64_t* __restrict__ ukeys, int* __restrict__ cstart, int* __restrict__ ncells) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int c = cell_of[j] - 1;
  cell_of[j] = c;
  if (j == 0 || keys[j] != keys[j - 1]) {
    ukeys[c] = keys[j];
    cstart[c] = j;
  }
  if (j == n - 1) {
    *ncells = c + 1;
    cstart[c + 1] = n;
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

// ---- DBSCAN ---------------------------------------------------------------------------------------------------------
// Union-find over input indices.  parent[i] <= i always holds (a root is only ever hooked under a smaller root), so the
// root of a component is its smallest core index whatever order the CAS operations land in.
__device__ __forceinline__ int find_root(volatile int* parent, int i) {
  int cur = parent[i];
  if (cur != i) {
    int prev = i, next;
    while (cur > (next = parent[cur])) {  // path halving; a stale read only sees a larger (still valid) ancestor
      parent[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

__device__ __forceinline__ void unite(int* parent, int a, int b) {
  int ra = find_root(parent, a), rb = find_root(parent, b);
  while (ra != rb) {
    const int lo = min(ra, rb), hi = max(ra, rb);
    const int old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) return;
    ra = find_root(parent, old);
    rb = find_root(parent, lo);
  }
}

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

// ---- host side ------------------------------------------------------------------------------------------------------
int blocks_for(long long n) { return (int)((n + kThreads - 1) / kThreads); }

// Caller-owned device scratch, carved in a fixed order (base == nullptr: sizes only).
struct Scratch {
  uint64_t* keys_in;
  uint64_t* keys;
  int* idx_in;
  int* perm;
  double* x;
  double* y;
  double* z;
  int* cell_of;
  uint64_t* ukeys;
  int* cstart;  // [n + 1]
  int* ncells;
  int* core;
  int* cmin;
  int* parent;
  int* flag;
  int* cid;
  void* cub;
  size_t cub_bytes;
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

// Sorted cell keys, sorted coordinates, cells and their first positions for cell side h and origin lo.
int build_grid(const double* pts, int n, const double* lo, double h, const Scratch& s, cudaStream_t st, Grid* g) {
  cell_key_kernel<<<blocks_for(n), kThreads, 0, st>>>(pts, n, lo[0], lo[1], lo[2], h, s.keys_in, s.idx_in);
  if (int rc = check_launch("cell_key_kernel")) return rc;
  size_t tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceRadixSort::SortPairs(s.cub, tb, s.keys_in, s.keys, s.idx_in, s.perm, n, 0, 3 * kAxisBits, st),
                          "cub SortPairs (cell keys)"))
    return rc;
  gather_kernel<<<blocks_for(n), kThreads, 0, st>>>(pts, n, s.keys, s.perm, s.x, s.y, s.z, s.flag);
  if (int rc = check_launch("gather_kernel")) return rc;
  tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceScan::InclusiveSum(s.cub, tb, s.flag, s.cell_of, n, st), "cub InclusiveSum (cells)")) return rc;
  cells_kernel<<<blocks_for(n), kThreads, 0, st>>>(n, s.keys, s.cell_of, s.ukeys, s.cstart, s.ncells);
  if (int rc = check_launch("cells_kernel")) return rc;
  *g = Grid{n, s.keys, s.perm, s.x, s.y, s.z, s.cell_of, s.ukeys, s.cstart, s.ncells};
  return FNR_OK;
}

double cell_side(double r) { return kCellShrink * r / std::sqrt(3.0); }

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
  radius_count_kernel<<<blocks_for(n), kThreads, 0, st>>>(g, radius * radius, cap, counts, nullptr);
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
  voxel_mean_kernel<<<blocks_for(n), kThreads, 0, st>>>(g, out);
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
  const int nb = blocks_for(n);
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
  const int nb = blocks_for(n);
  label_key_kernel<<<nb, kThreads, 0, st>>>(labels, n, K, kin, s.idx_in);
  if (int rc = check_launch("label_key_kernel")) return rc;
  int bits = 1;
  while (bits < 32 && (1ull << bits) <= (unsigned long long)K) ++bits;  // keys are 0..K
  size_t tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceRadixSort::SortPairs(s.cub, tb, kin, kout, s.idx_in, s.perm, n, 0, bits, st), "cub SortPairs (labels)"))
    return rc;
  for (int* b : {s.cstart, s.cell_of}) {  // an id no point carries sums to zero
    fill_kernel<<<blocks_for(K), kThreads, 0, st>>>(b, K, 0);
    if (int rc = check_launch("fill_kernel")) return rc;
  }
  segment_bounds_kernel<<<nb, kThreads, 0, st>>>(n, kout, s.cstart, s.cell_of);
  if (int rc = check_launch("segment_bounds_kernel")) return rc;
  cluster_sums_kernel<<<std::min(K, 8 * sm_count()), kThreads, 0, st>>>(points, s.perm, s.cstart, s.cell_of, K, sums, counts);
  return check_launch("cluster_sums_kernel");
}

}  // extern "C"
