// The sorted uniform grid of the point-cloud kernels (fnr_cluster.cu: neighbour queries; fnr_poisson.cu: the Poisson
// splat and its point-sample operator).  Cell keys (21 bits per axis, x-major, so key order is the C order of the cells)
// are radix-sorted with CUB, the points are gathered in key order -- a stable sort: input order inside a cell -- and
// every occupied cell gets its first sorted position.
#pragma once
#include <cub/cub.cuh>
#include <climits>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kGridThreads = 256;
constexpr int kAxisBits = 21;
constexpr long long kAxisCells = 1LL << kAxisBits;
constexpr uint64_t kAxisMask = (uint64_t)kAxisCells - 1;

__device__ __forceinline__ uint64_t pack_key(long long x, long long y, long long z) {
  return ((uint64_t)x << (2 * kAxisBits)) | ((uint64_t)y << kAxisBits) | (uint64_t)z;
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

// The device buffers a grid is built in (caller-owned scratch).
struct GridBuffers {
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
  int* flag;
  void* cub;
  size_t cub_bytes;
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

__global__ void __launch_bounds__(kGridThreads) cell_key_kernel(const double* __restrict__ pts, int n, double ox, double oy, double oz,
                                                                double h, uint64_t* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* p = pts + 3 * (size_t)i;
  keys[i] = pack_key(axis_cell(p[0], ox, h), axis_cell(p[1], oy, h), axis_cell(p[2], oz, h));
  idx[i] = i;
}

// sorted coordinates + "first of its cell" flags (inclusive-scanned into cell_of afterwards)
__global__ void __launch_bounds__(kGridThreads) gather_kernel(const double* __restrict__ pts, int n, const uint64_t* __restrict__ keys,
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
__global__ void __launch_bounds__(kGridThreads) cells_kernel(int n, const uint64_t* __restrict__ keys, int* __restrict__ cell_of,
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

// CUB temporary storage build_grid needs for n points.
int grid_cub_bytes(int n, size_t* bytes) {
  size_t a = 0, c = 0;
  if (check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr, n),
                 "cub SortPairs (cell keys) size query") ||
      check_cuda(cub::DeviceScan::InclusiveSum(nullptr, c, (const int*)nullptr, (int*)nullptr, n), "cub InclusiveSum size query"))
    return FNR_ERR_CUDA;
  *bytes = a > c ? a : c;
  return FNR_OK;
}

// Sorted cell keys, sorted coordinates, cells and their first positions for cell side h and origin lo (n >= 1).
int build_grid(const double* pts, int n, const double* lo, double h, const GridBuffers& s, cudaStream_t st, Grid* g) {
  cell_key_kernel<<<grid_for(n, kGridThreads, INT_MAX), kGridThreads, 0, st>>>(pts, n, lo[0], lo[1], lo[2], h, s.keys_in, s.idx_in);
  if (int rc = check_launch("cell_key_kernel")) return rc;
  size_t tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceRadixSort::SortPairs(s.cub, tb, s.keys_in, s.keys, s.idx_in, s.perm, n, 0, 3 * kAxisBits, st),
                          "cub SortPairs (cell keys)"))
    return rc;
  gather_kernel<<<grid_for(n, kGridThreads, INT_MAX), kGridThreads, 0, st>>>(pts, n, s.keys, s.perm, s.x, s.y, s.z, s.flag);
  if (int rc = check_launch("gather_kernel")) return rc;
  tb = s.cub_bytes;
  if (int rc = check_cuda(cub::DeviceScan::InclusiveSum(s.cub, tb, s.flag, s.cell_of, n, st), "cub InclusiveSum (cells)")) return rc;
  cells_kernel<<<grid_for(n, kGridThreads, INT_MAX), kGridThreads, 0, st>>>(n, s.keys, s.cell_of, s.ukeys, s.cstart, s.ncells);
  if (int rc = check_launch("cells_kernel")) return rc;
  *g = Grid{n, s.keys, s.perm, s.x, s.y, s.z, s.cell_of, s.ukeys, s.cstart, s.ncells};
  return FNR_OK;
}

}  // namespace

}  // namespace fnr
