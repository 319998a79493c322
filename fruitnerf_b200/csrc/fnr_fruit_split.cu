// Stage 3 of the fruit count on the device: scaled point-to-point ICP, Ward sub-centres and Hausdorff distances, batched
// over the merged groups that are candidates for a split (clustering/clustering_base.py:261-429).  clustering.py's numpy
// code (icp_scaled, ward_cut_centres, hausdorff) is the oracle of every kernel here.
//
// fp64 throughout.  Distances are (dx*dx + dy*dy) + dz*dz and transforms ((T0 x + T1 y) + T2 z) + T3 with explicit
// round-to-nearest intrinsics (no FMA), the order of the numpy code.  One CTA per problem; every block reduction is a
// fixed tree (shuffle-down inside a warp, then the warps in index order), so repeated runs give the same bits.  The
// caller owns every buffer and nothing synchronises the host.
#include <math_constants.h>
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxIcpTargets = 4096;
constexpr int kMaxIcpSource = 16384;
constexpr int kMaxWardPoints = 4096;
constexpr int kMaxTop = 5;     // merges undone by the k = 6 cut
constexpr int kCutRows = 20;   // 2 + 3 + 4 + 5 + 6 sub-centres
constexpr int kTile = 1024;    // Hausdorff: points of the scanned set staged per tile (24 KB)

// row r of the 3x4 transform T applied to (x, y, z)
__device__ __forceinline__ double affine_row(const double* T, int r, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * r], x), __dmul_rn(T[4 * r + 1], y)), __dmul_rn(T[4 * r + 2], z)), T[4 * r + 3]);
}

// Sums V values over the block with a fixed tree; afterwards out[0..V) holds the totals for every thread.
template <int V>
__device__ __forceinline__ void block_sum(const double (&v)[V], double* red, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    double x = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = __dadd_rn(x, __shfl_down_sync(0xffffffffu, x, o));
    if (lane == 0) red[warp * V + k] = x;
  }
  __syncthreads();
  if (threadIdx.x < V) {
    double s = red[threadIdx.x];
    for (int w = 1; w < kWarps; ++w) s = __dadd_rn(s, red[w * V + threadIdx.x]);
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// ---- ICP ------------------------------------------------------------------------------------------------------------
// One-sided Jacobi SVD of a 3x3 matrix: a = u diag(s) v^T, s descending.  Returns false when the rank is below 2 (the
// rotation is then not determined).
__device__ bool svd3(const double (&m)[3][3], double (&u)[3][3], double (&s)[3], double (&v)[3][3]) {
  double a[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      a[r][c] = m[r][c];
      v[r][c] = r == c ? 1.0 : 0.0;
    }
  for (int sweep = 0; sweep < 32; ++sweep) {
    bool rotated = false;
    for (int pair = 0; pair < 3; ++pair) {
      const int p = pair == 2 ? 1 : 0, q = pair == 0 ? 1 : 2;
      double al = 0.0, be = 0.0, ga = 0.0;
      for (int r = 0; r < 3; ++r) {
        al += a[r][p] * a[r][p];
        be += a[r][q] * a[r][q];
        ga += a[r][p] * a[r][q];
      }
      if (ga == 0.0 || fabs(ga) <= 1e-15 * sqrt(al * be)) continue;
      rotated = true;
      const double zeta = (be - al) / (2.0 * ga);
      const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
      for (int r = 0; r < 3; ++r) {
        const double ap = a[r][p], aq = a[r][q];
        a[r][p] = c * ap - sn * aq;
        a[r][q] = sn * ap + c * aq;
        const double vp = v[r][p], vq = v[r][q];
        v[r][p] = c * vp - sn * vq;
        v[r][q] = sn * vp + c * vq;
      }
    }
    if (!rotated) break;
  }
  for (int c = 0; c < 3; ++c) s[c] = sqrt(a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c]);
  for (int i = 0; i < 2; ++i)  // sort the columns by singular value, descending
    for (int j = 0; j < 2 - i; ++j)
      if (s[j] < s[j + 1]) {
        const double ts = s[j];
        s[j] = s[j + 1];
        s[j + 1] = ts;
        for (int r = 0; r < 3; ++r) {
          double t = a[r][j];
          a[r][j] = a[r][j + 1];
          a[r][j + 1] = t;
          t = v[r][j];
          v[r][j] = v[r][j + 1];
          v[r][j + 1] = t;
        }
      }
  if (!(s[1] > 1e-12 * s[0])) return false;
  for (int c = 0; c < 2; ++c)
    for (int r = 0; r < 3; ++r) u[r][c] = a[r][c] / s[c];
  if (s[2] > 1e-12 * s[0]) {
    for (int r = 0; r < 3; ++r) u[r][2] = a[r][2] / s[2];
  } else {  // rank 2: the third left vector completes a right-handed basis
    u[0][2] = u[1][0] * u[2][1] - u[2][0] * u[1][1];
    u[1][2] = u[2][0] * u[0][1] - u[0][0] * u[2][1];
    u[2][2] = u[0][0] * u[1][1] - u[1][0] * u[0][1];
  }
  return true;
}

__device__ __forceinline__ double det3(const double (&m)[3][3]) {
  return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
         m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}

// Eigen::umeyama(p, q, with_scaling = true) from the pair sums: tot[0..8] = sum (q - q_mean)(p - p_mean)^T row-major,
// tot[9] = sum |p - p_mean|^2.  Left-multiplies the update onto T (3x4).  A degenerate problem leaves T unchanged.
__device__ void umeyama_update(const double* tot, double cnt, const double (&mp)[3], const double (&mq)[3], double* T) {
  const double var = tot[9] / cnt;
  if (!(var > 0.0)) return;
  double sig[3][3], u[3][3], s[3], v[3][3];
  for (int k = 0; k < 9; ++k) sig[k / 3][k % 3] = tot[k] / cnt;
  if (!svd3(sig, u, s, v)) return;
  const double d = det3(u) * det3(v) < 0.0 ? -1.0 : 1.0;
  const double c = (s[0] + s[1] + d * s[2]) / var;
  double U[3][4];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) U[i][j] = c * (u[i][0] * v[j][0] + u[i][1] * v[j][1] + d * u[i][2] * v[j][2]);
  for (int i = 0; i < 3; ++i) U[i][3] = mq[i] - (U[i][0] * mp[0] + U[i][1] * mp[1] + U[i][2] * mp[2]);
  double N[12];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) N[4 * i + j] = U[i][0] * T[j] + U[i][1] * T[4 + j] + U[i][2] * T[8 + j] + (j == 3 ? U[i][3] : 0.0);
  for (int k = 0; k < 12; ++k) T[k] = N[k];
}

struct IcpArgs {
  const double* source;  // [m,3], shared by all problems
  int m;
  const double* targets;  // [*,3], problem b's targets are rows target_offsets[b] .. target_offsets[b+1]
  const int64_t* target_offsets;
  int max_targets;
  const double* init_translation;  // [B,3]
  double max_d2;
  int max_iteration;
  double relative_fitness, relative_rmse;
  double* transforms;  // [B,4,4]
  double* fitness;
  double* rmse;
  int32_t* iterations;
};

// One CTA per problem: the targets in shared memory, every transformed source point pairs with its nearest target by
// brute force (lowest index on ties) when the squared distance is < max_d2.
__global__ void __launch_bounds__(kThreads) icp_kernel(IcpArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* tx = reinterpret_cast<double*>(smem);
  double* ty = tx + a.max_targets;
  double* tz = ty + a.max_targets;
  int* corr = reinterpret_cast<int*>(tz + a.max_targets);
  __shared__ double red[kWarps * 10];
  __shared__ double tot[10];
  __shared__ double T[12];
  const int b = blockIdx.x, tid = threadIdx.x;
  const long long beg = a.target_offsets[b], n64 = a.target_offsets[b + 1] - beg;
  double* Tout = a.transforms + 16 * (size_t)b;
  if (n64 < 1 || n64 > a.max_targets) {  // refused: NaN transform, iteration count -1
    if (tid < 16) Tout[tid] = CUDART_NAN;
    if (tid == 0) {
      a.fitness[b] = a.rmse[b] = CUDART_NAN;
      a.iterations[b] = -1;
    }
    return;
  }
  const int n = (int)n64;
  for (int j = tid; j < n; j += kThreads) {
    const double* q = a.targets + 3 * (size_t)(beg + j);
    tx[j] = q[0];
    ty[j] = q[1];
    tz[j] = q[2];
  }
  if (tid < 12) T[tid] = (tid & 3) == 3 ? a.init_translation[3 * b + (tid >> 2)] : ((tid >> 2) == (tid & 3) ? 1.0 : 0.0);
  __syncthreads();

  // pairs of the current T; tot = {pairs, sum d2, sum p (3), sum q (3)}
  auto correspond = [&]() {
    double v[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = tid; i < a.m; i += kThreads) {
      const double* s = a.source + 3 * (size_t)i;
      const double px = affine_row(T, 0, s[0], s[1], s[2]), py = affine_row(T, 1, s[0], s[1], s[2]), pz = affine_row(T, 2, s[0], s[1], s[2]);
      double best = CUDART_INF;
      int bj = -1;
      for (int j = 0; j < n; ++j) {
        const double d = dist2(px, py, pz, tx[j], ty[j], tz[j]);
        if (d < best) {
          best = d;
          bj = j;
        }
      }
      if (best < a.max_d2) {
        corr[i] = bj;
        v[0] += 1.0;
        v[1] = __dadd_rn(v[1], best);
        v[2] = __dadd_rn(v[2], px);
        v[3] = __dadd_rn(v[3], py);
        v[4] = __dadd_rn(v[4], pz);
        v[5] = __dadd_rn(v[5], tx[bj]);
        v[6] = __dadd_rn(v[6], ty[bj]);
        v[7] = __dadd_rn(v[7], tz[bj]);
      } else {
        corr[i] = -1;
      }
    }
    block_sum<8>(v, red, tot);
  };

  correspond();
  double cnt = tot[0];
  double fit = cnt > 0.0 ? cnt / a.m : 0.0, err = cnt > 0.0 ? sqrt(tot[1] / cnt) : 0.0;
  int it = 0;
  while (it < a.max_iteration) {
    if (cnt >= 3.0) {  // fewer pairs: the update is the identity
      const double mp[3] = {tot[2] / cnt, tot[3] / cnt, tot[4] / cnt}, mq[3] = {tot[5] / cnt, tot[6] / cnt, tot[7] / cnt};
      double w[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      for (int i = tid; i < a.m; i += kThreads) {
        const int j = corr[i];
        if (j < 0) continue;
        const double* s = a.source + 3 * (size_t)i;
        const double pd[3] = {affine_row(T, 0, s[0], s[1], s[2]) - mp[0], affine_row(T, 1, s[0], s[1], s[2]) - mp[1],
                              affine_row(T, 2, s[0], s[1], s[2]) - mp[2]};
        const double qd[3] = {tx[j] - mq[0], ty[j] - mq[1], tz[j] - mq[2]};
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) w[3 * r + c] = __dadd_rn(w[3 * r + c], __dmul_rn(qd[r], pd[c]));
        w[9] = __dadd_rn(w[9], __dadd_rn(__dadd_rn(__dmul_rn(pd[0], pd[0]), __dmul_rn(pd[1], pd[1])), __dmul_rn(pd[2], pd[2])));
      }
      __shared__ double cov[10];
      block_sum<10>(w, red, cov);
      if (tid == 0) umeyama_update(cov, cnt, mp, mq, T);
      __syncthreads();
    }
    correspond();
    ++it;
    cnt = tot[0];
    const double f = cnt > 0.0 ? cnt / a.m : 0.0, e = cnt > 0.0 ? sqrt(tot[1] / cnt) : 0.0;
    const bool done = fabs(fit - f) < a.relative_fitness && fabs(err - e) < a.relative_rmse;
    fit = f;
    err = e;
    if (done) break;
  }
  if (tid < 16) Tout[tid] = tid < 12 ? T[tid] : (tid == 15 ? 1.0 : 0.0);
  if (tid == 0) {
    a.fitness[b] = fit;
    a.rmse[b] = err;
    a.iterations[b] = it;
  }
}

// ---- Ward -----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double ward_dist(double na, double nb, double dx, double dy, double dz) {
  const double w = __ddiv_rn(__dmul_rn(__dmul_rn(2.0, na), nb), __dadd_rn(na, nb));
  return __dmul_rn(__dsqrt_rn(w), __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))));
}

// The subtrees under merge m: for each of its slots, the latest earlier merge that kept that slot (none: a leaf).
__device__ int ward_children(const short2* rec, int m, int* out) {
  int k = 0;
  const int slots[2] = {rec[m].x, rec[m].y};
  for (int s = 0; s < 2; ++s)
    for (int j = m - 1; j >= 0; --j)
      if (rec[j].x == slots[s]) {
        out[k++] = j;
        break;
      }
  return k;
}

// One CTA per segment.  Clusters live in slots 0..n-1 (slot i starts as point i); a merge keeps the lower slot, so a
// cluster's slot is its smallest point index and slot 0 is never retired.  Nearest-neighbour chain: the chain's top a
// finds its nearest active cluster b by a block-wide argmin (ties: the chain's predecessor, then the lower slot); when b
// is the predecessor the two merge, else b is pushed.
__global__ void __launch_bounds__(kThreads) ward_kernel(const double* __restrict__ pts, const int64_t* __restrict__ offsets, int max_points,
                                                        double* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* cx = reinterpret_cast<double*>(smem);
  double* cy = cx + max_points;
  double* cz = cy + max_points;
  double* height = cz + max_points;
  int* size = reinterpret_cast<int*>(height + max_points);
  int* chain = size + max_points;  // the chain, then the parent slots of the base cut
  short2* rec = reinterpret_cast<short2*>(chain + max_points);  // (slot_lo, slot_hi) of merge m
  __shared__ double rd[kWarps];
  __shared__ int ri[kWarps];
  __shared__ int s_len, s_merged, s_ntop, s_top[kMaxTop], s_base[kMaxTop + 1];
  __shared__ double red[kWarps * 4 * (kMaxTop + 1)];
  __shared__ double sums[4 * (kMaxTop + 1)];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long beg = offsets[b], n64 = offsets[b + 1] - beg;
  double* o = out + 3 * kCutRows * (size_t)b;
  for (int k = tid; k < 3 * kCutRows; k += kThreads) o[k] = CUDART_NAN;  // rows no cut reaches stay NaN
  if (n64 < 1 || n64 > max_points) return;
  const int n = (int)n64;
  for (int i = tid; i < n; i += kThreads) {
    const double* p = pts + 3 * (size_t)(beg + i);
    cx[i] = p[0];
    cy[i] = p[1];
    cz[i] = p[2];
    size[i] = 1;
  }
  if (tid == 0) {
    s_len = 0;
    s_merged = 0;
  }
  __syncthreads();
  while (s_merged < n - 1) {
    if (tid == 0 && s_len == 0) chain[s_len++] = 0;
    __syncthreads();
    const int len = s_len, ca = chain[len - 1];
    const double ax = cx[ca], ay = cy[ca], az = cz[ca], na = (double)size[ca];
    double best = CUDART_INF;
    int bi = 0x7fffffff;
    for (int j = tid; j < n; j += kThreads) {
      if (j == ca || size[j] == 0) continue;
      const double d = ward_dist(na, (double)size[j], cx[j] - ax, cy[j] - ay, cz[j] - az);
      if (d < best) {
        best = d;
        bi = j;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double od = __shfl_down_sync(0xffffffffu, best, off);
      const int oi = __shfl_down_sync(0xffffffffu, bi, off);
      if (od < best || (od == best && oi < bi)) {
        best = od;
        bi = oi;
      }
    }
    if (lane == 0) {
      rd[warp] = best;
      ri[warp] = bi;
    }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kWarps; ++w)
        if (rd[w] < best || (rd[w] == best && ri[w] < bi)) {
          best = rd[w];
          bi = ri[w];
        }
      const int prev = len >= 2 ? chain[len - 2] : -1;
      if (prev >= 0 && ward_dist(na, (double)size[prev], cx[prev] - ax, cy[prev] - ay, cz[prev] - az) == best) bi = prev;
      if (bi == prev) {
        const int lo = min(ca, prev), hi = max(ca, prev), m = s_merged;
        const double nl = (double)size[lo], nh = (double)size[hi], ns = __dadd_rn(nl, nh);
        cx[lo] = __ddiv_rn(__dadd_rn(__dmul_rn(nl, cx[lo]), __dmul_rn(nh, cx[hi])), ns);
        cy[lo] = __ddiv_rn(__dadd_rn(__dmul_rn(nl, cy[lo]), __dmul_rn(nh, cy[hi])), ns);
        cz[lo] = __ddiv_rn(__dadd_rn(__dmul_rn(nl, cz[lo]), __dmul_rn(nh, cz[hi])), ns);
        size[lo] += size[hi];
        size[hi] = 0;
        rec[m] = make_short2((short)lo, (short)hi);
        height[m] = best;
        s_merged = m + 1;
        s_len = len - 2;
      } else {
        chain[len] = bi;
        s_len = len + 1;
      }
    }
    __syncthreads();
  }

  // The cut at k undoes the k - 1 highest merges, taken top-down: the root (the last merge), then repeatedly the highest
  // (height, then later merge) of the merges directly below those taken.
  if (tid == 0) {
    int ntop = 0, frontier[2 * kMaxTop + 2], nf = 0;
    if (n > 1) {
      s_top[ntop++] = n - 2;
      nf = ward_children(rec, n - 2, frontier);
    }
    while (ntop < kMaxTop && nf > 0) {
      int pick = 0;
      for (int f = 1; f < nf; ++f)
        if (height[frontier[f]] > height[frontier[pick]] || (height[frontier[f]] == height[frontier[pick]] && frontier[f] > frontier[pick])) pick = f;
      const int m = frontier[pick];
      frontier[pick] = frontier[--nf];
      s_top[ntop++] = m;
      nf += ward_children(rec, m, frontier + nf);
    }
    s_ntop = ntop;
    // base clusters of the deepest cut: slot 0 and the upper slot of every merge undone, in slot order
    int nb = 0;
    s_base[nb++] = 0;
    for (int t = 0; t < ntop; ++t) {
      int v = rec[s_top[t]].y, p = nb++;
      while (p > 0 && s_base[p - 1] > v) {
        s_base[p] = s_base[p - 1];
        --p;
      }
      s_base[p] = v;
    }
  }
  __syncthreads();
  const int ntop = s_ntop, nbase = ntop + 1;
  for (int i = tid; i < n; i += kThreads) chain[i] = i;
  __syncthreads();
  if (tid == 0) {
    for (int m = 0; m < n - 1; ++m) {
      bool undone = false;
      for (int t = 0; t < ntop; ++t) undone |= s_top[t] == m;
      if (!undone) chain[rec[m].y] = rec[m].x;
    }
    for (int i = 1; i < n; ++i) chain[i] = chain[chain[i]];  // parent < child: one pass in slot order finds every root
  }
  __syncthreads();
  double v[4 * (kMaxTop + 1)];
#pragma unroll
  for (int k = 0; k < 4 * (kMaxTop + 1); ++k) v[k] = 0.0;
  for (int i = tid; i < n; i += kThreads) {
    const int r = chain[i];
    const double* p = pts + 3 * (size_t)(beg + i);
#pragma unroll
    for (int c = 0; c < kMaxTop + 1; ++c)
      if (c < nbase && s_base[c] == r) {
        v[4 * c] = __dadd_rn(v[4 * c], p[0]);
        v[4 * c + 1] = __dadd_rn(v[4 * c + 1], p[1]);
        v[4 * c + 2] = __dadd_rn(v[4 * c + 2], p[2]);
        v[4 * c + 3] += 1.0;
      }
  }
  block_sum<4 * (kMaxTop + 1)>(v, red, sums);
  if (tid == 0) {
    int slot[kMaxTop + 1], live = nbase;
    double s[kMaxTop + 1][4];
    for (int c = 0; c < nbase; ++c) {
      slot[c] = s_base[c];
      for (int k = 0; k < 4; ++k) s[c][k] = sums[4 * c + k];
    }
    const int row0[kMaxTop + 1] = {0, 0, 2, 5, 9, 14};  // first row of the cut with k clusters
    for (int k = nbase; k >= 2; --k) {
      for (int c = 0; c < k; ++c)
        for (int d = 0; d < 3; ++d) o[3 * (row0[k - 1] + c) + d] = s[c][d] / s[c][3];
      const int lo = rec[s_top[k - 2]].x, hi = rec[s_top[k - 2]].y;
      int clo = 0, chi = 0;
      for (int c = 0; c < live; ++c) {
        if (slot[c] == lo) clo = c;
        if (slot[c] == hi) chi = c;
      }
      for (int d = 0; d < 4; ++d) s[clo][d] += s[chi][d];
      for (int c = chi; c + 1 < live; ++c) {
        slot[c] = slot[c + 1];
        for (int d = 0; d < 4; ++d) s[c][d] = s[c + 1][d];
      }
      --live;
    }
  }
}

// ---- Hausdorff ------------------------------------------------------------------------------------------------------
// One CTA per pair: each thread takes query points of one set in turn, scans the other set through shared-memory tiles
// and keeps the largest nearest squared distance; the block maximum (exact, so order-free) gives sqrt(max) at the end.
__global__ void __launch_bounds__(kThreads) hausdorff_kernel(const double* __restrict__ a, const int64_t* __restrict__ a_ranges,
                                                             const double* __restrict__ b, const int64_t* __restrict__ b_ranges,
                                                             double* __restrict__ out) {
  __shared__ double sx[kTile], sy[kTile], sz[kTile];
  __shared__ double red[kWarps];
  const int pair = blockIdx.x, tid = threadIdx.x;
  const long long ab = a_ranges[2 * pair], ae = a_ranges[2 * pair + 1], bb = b_ranges[2 * pair], be = b_ranges[2 * pair + 1];
  if (!(ae > ab && be > bb)) {
    if (tid == 0) out[pair] = CUDART_NAN;
    return;
  }
  double worst = 0.0;
  for (int dir = 0; dir < 2; ++dir) {
    const double* P = dir == 0 ? a : b;
    const double* Q = dir == 0 ? b : a;
    const long long pb = dir == 0 ? ab : bb, pe = dir == 0 ? ae : be, qb = dir == 0 ? bb : ab, qe = dir == 0 ? be : ae;
    for (long long base = pb; base < pe; base += kThreads) {
      const long long i = base + tid;
      const bool valid = i < pe;
      double px = 0.0, py = 0.0, pz = 0.0, best = CUDART_INF;
      if (valid) {
        px = P[3 * i];
        py = P[3 * i + 1];
        pz = P[3 * i + 2];
      }
      for (long long t = qb; t < qe; t += kTile) {
        const int cnt = (int)min((long long)kTile, qe - t);
        __syncthreads();
        for (int j = tid; j < cnt; j += kThreads) {
          sx[j] = Q[3 * (t + j)];
          sy[j] = Q[3 * (t + j) + 1];
          sz[j] = Q[3 * (t + j) + 2];
        }
        __syncthreads();
        if (valid)
          for (int j = 0; j < cnt; ++j) best = fmin(best, dist2(px, py, pz, sx[j], sy[j], sz[j]));
      }
      if (valid) worst = fmax(worst, best);
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) worst = fmax(worst, __shfl_down_sync(0xffffffffu, worst, off));
  if ((tid & 31) == 0) red[tid >> 5] = worst;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < kWarps; ++w) worst = fmax(worst, red[w]);
    out[pair] = __dsqrt_rn(worst);
  }
}

size_t icp_smem(int max_targets, int m) { return (size_t)max_targets * 3 * sizeof(double) + (size_t)m * sizeof(int); }

size_t ward_smem(int max_points) { return (size_t)max_points * (4 * sizeof(double) + 2 * sizeof(int) + sizeof(short2)); }

int set_smem(const void* kernel, size_t bytes, const char* what) {
  return check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), what);
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_icp_scaled(const double* source, int32_t num_source, const double* targets, const int64_t* target_offsets, int32_t num_problems,
                   int32_t max_targets, const double* init_translation, double max_distance, int32_t max_iteration,
                   double relative_fitness, double relative_rmse, double* transforms, double* fitness, double* rmse, int32_t* iterations,
                   void* stream) {
  const char* what = "fnr_icp_scaled";
  if (num_problems < 0 || num_source < 1 || max_targets < 1 || max_iteration < 0 || !(max_distance > 0.0) || !std::isfinite(max_distance) ||
      !(relative_fitness >= 0.0) || !(relative_rmse >= 0.0) ||
      (num_problems > 0 && (!source || !targets || !target_offsets || !init_translation || !transforms || !fitness || !rmse || !iterations))) {
    set_error("%s: invalid arguments (problems %d, source points %d, max targets %d, max_distance %g, max_iteration %d)", what, num_problems,
              num_source, max_targets, max_distance, max_iteration);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (max_targets > kMaxIcpTargets || num_source > kMaxIcpSource) {
    set_error("%s: %d targets per problem and %d source points; at most %d and %d are supported", what, max_targets, num_source, kMaxIcpTargets,
              kMaxIcpSource);
    return FNR_ERR_UNSUPPORTED;
  }
  if (num_problems == 0) return FNR_OK;
  const size_t smem = icp_smem(max_targets, num_source);
  if (int rc = set_smem((const void*)icp_kernel, smem, "fnr_icp_scaled (shared memory)")) return rc;
  IcpArgs a{source, num_source, targets, target_offsets, max_targets, init_translation, max_distance * max_distance, max_iteration,
            relative_fitness, relative_rmse, transforms, fitness, rmse, iterations};
  icp_kernel<<<num_problems, kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return check_launch("icp_kernel");
}

int fnr_ward_cut(const double* points, const int64_t* offsets, int32_t num_segments, int32_t max_points, double* centres, void* stream) {
  const char* what = "fnr_ward_cut";
  if (num_segments < 0 || max_points < 1 || (num_segments > 0 && (!points || !offsets || !centres))) {
    set_error("%s: invalid arguments (segments %d, max points %d)", what, num_segments, max_points);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (max_points > kMaxWardPoints) {
    set_error("%s: %d points per segment; at most %d are supported", what, max_points, kMaxWardPoints);
    return FNR_ERR_UNSUPPORTED;
  }
  if (num_segments == 0) return FNR_OK;
  const size_t smem = ward_smem(max_points);
  if (int rc = set_smem((const void*)ward_kernel, smem, "fnr_ward_cut (shared memory)")) return rc;
  ward_kernel<<<num_segments, kThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(points, offsets, max_points, centres);
  return check_launch("ward_kernel");
}

int fnr_hausdorff(const double* a, const int64_t* a_ranges, const double* b, const int64_t* b_ranges, int32_t num_pairs, double* distances,
                  void* stream) {
  const char* what = "fnr_hausdorff";
  if (num_pairs < 0 || (num_pairs > 0 && (!a || !a_ranges || !b || !b_ranges || !distances))) {
    set_error("%s: invalid arguments (pairs %d)", what, num_pairs);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (num_pairs == 0) return FNR_OK;
  hausdorff_kernel<<<num_pairs, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a, a_ranges, b, b_ranges, distances);
  return check_launch("hausdorff_kernel");
}

}  // extern "C"
