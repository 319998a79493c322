// Screened Poisson surface reconstruction on a dense grid (`ns-export-semantics poisson`, nerfstudio ns-export poisson /
// open3d create_from_point_cloud_poisson; DESIGN section 4.3m).  The points' cube (the bounding box's largest side
// scaled about its centre) carries R = 2^d cells per axis, h = 1/R in cube units, and a trilinear hat per node.
//   poisson_check_kernel   refuses non-finite points and points outside the cube (one device flag, read by the host)
//   frac_kernel / cell_map_kernel  the sorted uniform grid of fnr_grid.cuh at cell side = side / R: each sorted point's
//                          position in its cell, and a dense map from cell to occupied-cell index
//   splat_kernel           per node, a gather over the points of its 8 adjacent cells (cell order, then input order) of
//                          density, normal field, colour and fruit sums and of sum phi^2 (the screening diagonal), in fp64,
//                          rounded to fp32 once.  No atomics: every run gives the same bits, and poisson.restated_splat
//                          reproduces them.
//   rhs_kernel             b_i = sum_j (int grad phi_i phi_j) . v_j, the Q1 27-point stencil in a fixed order
//   apply_kernel           y = (K + alpha a S^T S) x: the Q1 stiffness stencil (cells inside the cube only: Neumann
//                          boundaries) plus the point samples S x gathered back by node
//   CG kernels             Jacobi-preconditioned conjugate gradient in fp32 with fp64 block-partial dot products (a fixed
//                          number of blocks, reduced in a fixed order), coarse-to-fine over depths max(d-3, 4)..d
// The 1D factors of the stencils: mass M1 (h/3 at an end node, 2h/3 inside, h/6 off the diagonal), stiffness K1 (1/h,
// 2/h, -1/h) and the gradient-mass G1[i][j] = int phi_i' phi_j (-1/2 at node 0, +1/2 at node R, 0 inside; -1/2 to the
// right, +1/2 to the left).  K = K1xM1xM1 + M1xK1xM1 + M1xM1xK1 and G_x = G1xM1xM1 etc., which is the assembly of the
// 8x8 Q1 element matrices over the R^3 cells (poisson.assemble).
#include <algorithm>
#include <climits>
#include <cmath>
#include "fnr_common.cuh"
#include "fnr_grid.cuh"
#include "fnr_kernels.h"

namespace fnr {

namespace {

constexpr int kThreads = 256;
constexpr int kRedBlocks = 1024;  // blocks of every reduction kernel: partial sums in a fixed order
constexpr int kMaxDepth = 10;

struct Level {
  int d;
  long long R, Nn, M;  // cells per axis, nodes per axis, nodes
  double o[3], hw;     // cube origin and world cell side
  double h;            // cube-unit cell side 1/R
  double m_off, m_end, m_mid, k_off, k_end, k_mid;  // the 1D factors: h/6, h/3, 2h/3, -1/h, 1/h, 2/h
};

Level make_level(int d, const double* origin, double side) {
  Level L;
  L.d = d;
  L.R = 1LL << d;
  L.Nn = L.R + 1;
  L.M = L.Nn * L.Nn * L.Nn;
  for (int a = 0; a < 3; ++a) L.o[a] = origin[a];
  L.hw = side / (double)L.R;
  L.h = 1.0 / (double)L.R;
  L.m_off = L.h / 6.0;
  L.m_end = L.h / 3.0;
  L.m_mid = (2.0 * L.h) / 3.0;
  L.k_off = -1.0 / L.h;
  L.k_end = 1.0 / L.h;
  L.k_mid = 2.0 / L.h;
  return L;
}

struct Sorted {  // the points in cell order
  int n;
  const int* perm;          // [n] input index
  const uint64_t* keys;     // [n] cell key
  const double* t;          // [n,3] position inside the cell, [0,1)
  const int* cstart;        // [ncells + 1]
  const int* cell_map;      // [R^3] occupied-cell index or -1
};

// 1D factors at node I (0..R) for the neighbour I + o, o in {-1, 0, 1} (the values are computed once, in make_level)
__device__ __forceinline__ double m1(const Level& L, long long I, int o) {
  if (I + o < 0 || I + o > L.R) return 0.0;
  if (o) return L.m_off;
  return (I == 0 || I == L.R) ? L.m_end : L.m_mid;
}
__device__ __forceinline__ double k1(const Level& L, long long I, int o) {
  if (I + o < 0 || I + o > L.R) return 0.0;
  if (o) return L.k_off;
  return (I == 0 || I == L.R) ? L.k_end : L.k_mid;
}
__device__ __forceinline__ double g1(long long I, int o, long long R) {
  if (I + o < 0 || I + o > R) return 0.0;
  if (o) return o > 0 ? -0.5 : 0.5;
  return I == 0 ? -0.5 : (I == R ? 0.5 : 0.0);
}

__device__ __forceinline__ void node_ijk(long long i, long long Nn, long long& I, long long& J, long long& K) {
  K = i % Nn;
  const long long q = i / Nn;
  J = q % Nn;
  I = q / Nn;
}

// phi of the node at corner (bx, by, bz) of the cell holding sorted point j
__device__ __forceinline__ double corner_phi(const double* t, int bx, int by, int bz) {
  const double wx = bx ? t[0] : __dsub_rn(1.0, t[0]);
  const double wy = by ? t[1] : __dsub_rn(1.0, t[1]);
  const double wz = bz ? t[2] : __dsub_rn(1.0, t[2]);
  return __dmul_rn(__dmul_rn(wx, wy), wz);
}

// Calls f(j, phi_i(p_j)) for the points of node i's adjacent cells, in cell order, then sorted (= input) order.
template <class F>
__device__ __forceinline__ void for_each_node_point(const Sorted& S, const Level& L, long long I, long long J, long long K, F&& f) {
  for (int a = 0; a < 2; ++a) {
    const long long cx = I - 1 + a;
    if (cx < 0 || cx >= L.R) continue;
    for (int b = 0; b < 2; ++b) {
      const long long cy = J - 1 + b;
      if (cy < 0 || cy >= L.R) continue;
      for (int c = 0; c < 2; ++c) {
        const long long cz = K - 1 + c;
        if (cz < 0 || cz >= L.R) continue;
        const int id = __ldg(S.cell_map + (cx * L.R + cy) * L.R + cz);
        if (id < 0) continue;
        const int e = __ldg(S.cstart + id + 1);
        for (int j = __ldg(S.cstart + id); j < e; ++j) f(j, corner_phi(S.t + 3 * (size_t)j, 1 - a, 1 - b, 1 - c));
      }
    }
  }
}

// Deterministic fp64 block sum (blockDim.x == kThreads); thread 0 gets the result.
__device__ __forceinline__ double block_sum(double v, double* s_warp) {
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_warp[warp] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) r = __dadd_rn(r, s_warp[w]);
  return r;
}

// ---- validation and the sorted grid ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) poisson_check_kernel(const double* __restrict__ pts, long long n, Level L, int* __restrict__ bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    bool ok = true;
    for (int a = 0; a < 3; ++a) {
      const double p = pts[3 * i + a];
      if (!isfinite(p)) {
        ok = false;
        break;
      }
      const double c = floor(__ddiv_rn(__dsub_rn(p, L.o[a]), L.hw));
      ok = ok && c >= 0.0 && c <= (double)(L.R - 1);
    }
    if (!ok) atomicOr(bad, 1);
  }
}

__global__ void __launch_bounds__(kThreads) frac_kernel(Grid g, Level L, double* __restrict__ t) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= g.n) return;
  const uint64_t k = g.keys[j];
  const double p[3] = {g.x[j], g.y[j], g.z[j]};
  const long long c[3] = {(long long)(k >> (2 * kAxisBits)), (long long)((k >> kAxisBits) & kAxisMask), (long long)(k & kAxisMask)};
  for (int a = 0; a < 3; ++a) t[3 * (size_t)j + a] = __dsub_rn(__ddiv_rn(__dsub_rn(p[a], L.o[a]), L.hw), (double)c[a]);
}

__global__ void __launch_bounds__(kThreads) fill_int_kernel(int* __restrict__ a, long long n, int v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) a[i] = v;
}

__global__ void __launch_bounds__(kThreads) cell_map_kernel(Grid g, Level L, int* __restrict__ cell_map) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= *g.ncells) return;
  const uint64_t k = g.ukeys[c];
  const long long x = (long long)(k >> (2 * kAxisBits)), y = (long long)((k >> kAxisBits) & kAxisMask), z = (long long)(k & kAxisMask);
  cell_map[(x * L.R + y) * L.R + z] = c;
}

// a = h^2 * occupied cells / n (the area per sample) and the normal-field scale a / h^3
__global__ void area_kernel(const int* __restrict__ ncells, int n, Level L, double* __restrict__ scalars) {
  const double a = __ddiv_rn(__dmul_rn(__dmul_rn(L.h, L.h), (double)*ncells), (double)n);
  scalars[0] = a;
  scalars[1] = __ddiv_rn(a, __dmul_rn(__dmul_rn(L.h, L.h), L.h));
}

// ---- splat and right-hand side ---------------------------------------------------------------------------------------
struct KSplat {
  const float *normals, *colors, *fruit;  // input order; colors / fruit may be NULL
  const double* scalars;
  float *density, *vfield, *node_colors, *node_fruit, *ssq;  // density / colours / fruit may be NULL
};

__global__ void __launch_bounds__(kThreads) splat_kernel(Sorted S, Level L, KSplat A) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.M; i += (long long)gridDim.x * blockDim.x) {
    long long I, J, K;
    node_ijk(i, L.Nn, I, J, K);
    double rho = 0.0, nv[3] = {0.0, 0.0, 0.0}, col[3] = {0.0, 0.0, 0.0}, fr = 0.0, sq = 0.0;
    for_each_node_point(S, L, I, J, K, [&](int j, double phi) {
      const size_t p = (size_t)__ldg(S.perm + j);
      rho = __dadd_rn(rho, phi);
      sq = __dadd_rn(sq, __dmul_rn(phi, phi));
#pragma unroll
      for (int a = 0; a < 3; ++a) nv[a] = __dadd_rn(nv[a], __dmul_rn(phi, (double)__ldg(A.normals + 3 * p + a)));
      if (A.node_colors) {
#pragma unroll
        for (int a = 0; a < 3; ++a) col[a] = __dadd_rn(col[a], __dmul_rn(phi, (double)__ldg(A.colors + 3 * p + a)));
      }
      if (A.node_fruit) fr = __dadd_rn(fr, __dmul_rn(phi, (double)__ldg(A.fruit + p)));
    });
    const double scale = A.scalars[1];
    for (int a = 0; a < 3; ++a) A.vfield[3 * i + a] = (float)__dmul_rn(scale, nv[a]);
    if (A.density) A.density[i] = (float)rho;
    if (A.node_colors)
      for (int a = 0; a < 3; ++a) A.node_colors[3 * i + a] = rho > 0.0 ? (float)__ddiv_rn(col[a], rho) : 0.f;
    if (A.node_fruit) A.node_fruit[i] = rho > 0.0 ? (float)__ddiv_rn(fr, rho) : 0.f;
    A.ssq[i] = (float)sq;
  }
}

__global__ void __launch_bounds__(kThreads) rhs_kernel(Level L, const float* __restrict__ v, float* __restrict__ b) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.M; i += (long long)gridDim.x * blockDim.x) {
    long long I, J, K;
    node_ijk(i, L.Nn, I, J, K);
    double acc = 0.0;
    for (int dx = -1; dx <= 1; ++dx) {
      if (I + dx < 0 || I + dx > L.R) continue;
      const double mx = m1(L, I, dx), gx = g1(I, dx, L.R);
      for (int dy = -1; dy <= 1; ++dy) {
        if (J + dy < 0 || J + dy > L.R) continue;
        const double my = m1(L, J, dy), gy = g1(J, dy, L.R);
        for (int dz = -1; dz <= 1; ++dz) {
          if (K + dz < 0 || K + dz > L.R) continue;
          const double mz = m1(L, K, dz), gz = g1(K, dz, L.R);
          const float* vj = v + 3 * (i + (dx * L.Nn + dy) * L.Nn + dz);
          acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(__dmul_rn(gx, my), mz), (double)__ldg(vj)));
          acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(__dmul_rn(mx, gy), mz), (double)__ldg(vj + 1)));
          acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(__dmul_rn(mx, my), gz), (double)__ldg(vj + 2)));
        }
      }
    }
    b[i] = (float)acc;
  }
}

// ---- the operator ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ double stencil_k(const Level& L, long long i, long long I, long long J, long long K, const float* __restrict__ x) {
  double acc = 0.0;
  for (int dx = -1; dx <= 1; ++dx) {
    if (I + dx < 0 || I + dx > L.R) continue;
    const double mx = m1(L, I, dx), kx = k1(L, I, dx);
    for (int dy = -1; dy <= 1; ++dy) {
      if (J + dy < 0 || J + dy > L.R) continue;
      const double my = m1(L, J, dy), ky = k1(L, J, dy);
      for (int dz = -1; dz <= 1; ++dz) {
        if (K + dz < 0 || K + dz > L.R) continue;
        const double mz = m1(L, K, dz), kz = k1(L, K, dz);
        const double c = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(kx, my), mz), __dmul_rn(__dmul_rn(mx, ky), mz)), __dmul_rn(__dmul_rn(mx, my), kz));
        acc = __dadd_rn(acc, __dmul_rn(c, (double)__ldg(x + i + (dx * L.Nn + dy) * L.Nn + dz)));
      }
    }
  }
  return acc;
}

// S x: the grid sampled at every sorted point (fp64)
__global__ void __launch_bounds__(kThreads) point_sample_kernel(Sorted S, Level L, const float* __restrict__ x, double* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= S.n) return;
  const uint64_t k = S.keys[j];
  const long long c[3] = {(long long)(k >> (2 * kAxisBits)), (long long)((k >> kAxisBits) & kAxisMask), (long long)(k & kAxisMask)};
  const double* t = S.t + 3 * (size_t)j;
  double acc = 0.0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int bx = q & 1, by = (q >> 1) & 1, bz = (q >> 2) & 1;
    acc = __dadd_rn(acc, __dmul_rn(corner_phi(t, bx, by, bz), (double)__ldg(x + ((c[0] + bx) * L.Nn + c[1] + by) * L.Nn + c[2] + bz)));
  }
  out[j] = acc;
}

// y = K x + alpha a S^T (S x) (samples: S x from point_sample_kernel); with `partial`, per-block sums of x . y
__global__ void __launch_bounds__(kThreads) apply_kernel(Sorted S, Level L, const double* __restrict__ scalars, double alpha, const float* __restrict__ x,
                                                         const double* __restrict__ samples, float* __restrict__ y, double* __restrict__ partial) {
  __shared__ double s_warp[kThreads / 32];
  const double w = __dmul_rn(alpha, scalars[0]);
  double dot = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.M; i += (long long)gridDim.x * blockDim.x) {
    long long I, J, K;
    node_ijk(i, L.Nn, I, J, K);
    double st = 0.0;
    for_each_node_point(S, L, I, J, K, [&](int j, double phi) { st = __dadd_rn(st, __dmul_rn(phi, __ldg(samples + j))); });
    const float yi = (float)__dadd_rn(stencil_k(L, i, I, J, K, x), __dmul_rn(w, st));
    y[i] = yi;
    dot = __dadd_rn(dot, __dmul_rn((double)x[i], (double)yi));
  }
  if (partial) {
    const double s = block_sum(dot, s_warp);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
  }
}

// Jacobi diagonal: K_ii + alpha a sum phi_i^2
__global__ void __launch_bounds__(kThreads) diag_kernel(Level L, const double* __restrict__ scalars, double alpha, const float* __restrict__ ssq,
                                                        float* __restrict__ diag) {
  const double w = __dmul_rn(alpha, scalars[0]);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.M; i += (long long)gridDim.x * blockDim.x) {
    long long I, J, K;
    node_ijk(i, L.Nn, I, J, K);
    const double mx = m1(L, I, 0), my = m1(L, J, 0), mz = m1(L, K, 0);
    const double kii = __dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(k1(L, I, 0), my), mz), __dmul_rn(__dmul_rn(mx, k1(L, J, 0)), mz)),
                                 __dmul_rn(__dmul_rn(mx, my), k1(L, K, 0)));
    diag[i] = (float)__dadd_rn(kii, __dmul_rn(w, (double)ssq[i]));
  }
}

// ---- conjugate gradient ----------------------------------------------------------------------------------------------
struct Cg {  // device scalars
  double rz, rr, bb, alpha, beta;
};

// r = b - Ax, z = r / D, p = z; partial sums of r.z, r.r, b.b
__global__ void __launch_bounds__(kThreads) cg_init_kernel(long long M, const float* __restrict__ b, const float* __restrict__ ax,
                                                           const float* __restrict__ diag, float* __restrict__ r, float* __restrict__ z,
                                                           float* __restrict__ p, double* __restrict__ partial) {
  __shared__ double s_warp[kThreads / 32];
  double rz = 0.0, rr = 0.0, bb = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
    const float ri = __fsub_rn(b[i], ax[i]), zi = __fdiv_rn(ri, diag[i]);
    r[i] = ri;
    z[i] = zi;
    p[i] = zi;
    rz = __dadd_rn(rz, __dmul_rn((double)ri, (double)zi));
    rr = __dadd_rn(rr, __dmul_rn((double)ri, (double)ri));
    bb = __dadd_rn(bb, __dmul_rn((double)b[i], (double)b[i]));
  }
  const double s0 = block_sum(rz, s_warp), s1 = block_sum(rr, s_warp), s2 = block_sum(bb, s_warp);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s0;
    partial[kRedBlocks + blockIdx.x] = s1;
    partial[2 * kRedBlocks + blockIdx.x] = s2;
  }
}

// x += alpha p, r -= alpha Ap, z = r / D; partial sums of r.r and r.z
__global__ void __launch_bounds__(kThreads) cg_update_kernel(long long M, const Cg* __restrict__ cg, const float* __restrict__ p,
                                                             const float* __restrict__ ap, const float* __restrict__ diag, float* __restrict__ x,
                                                             float* __restrict__ r, float* __restrict__ z, double* __restrict__ partial) {
  __shared__ double s_warp[kThreads / 32];
  const float alpha = (float)cg->alpha;
  double rr = 0.0, rz = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x) {
    x[i] = __fadd_rn(x[i], __fmul_rn(alpha, p[i]));
    const float ri = __fsub_rn(r[i], __fmul_rn(alpha, ap[i])), zi = __fdiv_rn(ri, diag[i]);
    r[i] = ri;
    z[i] = zi;
    rr = __dadd_rn(rr, __dmul_rn((double)ri, (double)ri));
    rz = __dadd_rn(rz, __dmul_rn((double)ri, (double)zi));
  }
  const double s0 = block_sum(rr, s_warp), s1 = block_sum(rz, s_warp);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s0;
    partial[kRedBlocks + blockIdx.x] = s1;
  }
}

__global__ void __launch_bounds__(kThreads) cg_direction_kernel(long long M, const Cg* __restrict__ cg, const float* __restrict__ z, float* __restrict__ p) {
  const float beta = (float)cg->beta;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (long long)gridDim.x * blockDim.x)
    p[i] = __fadd_rn(z[i], __fmul_rn(beta, p[i]));
}

enum CgStep { kCgInit = 0, kCgAlpha = 1, kCgBeta = 2 };

// One block: the partial sums in a fixed order, then the scalar step.
__global__ void __launch_bounds__(kThreads) cg_scalars_kernel(const double* __restrict__ partial, int step, Cg* __restrict__ cg) {
  __shared__ double s_warp[kThreads / 32];
  double s[3];
  const int nk = step == kCgInit ? 3 : (step == kCgAlpha ? 1 : 2);
  for (int k = 0; k < nk; ++k) {
    double v = 0.0;
    for (int b = threadIdx.x; b < kRedBlocks; b += kThreads) v = __dadd_rn(v, partial[k * kRedBlocks + b]);
    s[k] = block_sum(v, s_warp);
  }
  if (threadIdx.x) return;
  if (step == kCgInit) {
    cg->rz = s[0];
    cg->rr = s[1];
    cg->bb = s[2];
  } else if (step == kCgAlpha) {
    cg->alpha = s[0] > 0.0 ? cg->rz / s[0] : 0.0;
  } else {
    cg->rr = s[0];
    cg->beta = cg->rz > 0.0 ? s[1] / cg->rz : 0.0;
    cg->rz = s[1];
  }
}

// trilinear prolongation of the depth d-1 grid xc to depth d
__global__ void __launch_bounds__(kThreads) prolong_kernel(Level L, const float* __restrict__ xc, float* __restrict__ xf) {
  const long long Nc = L.R / 2 + 1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.M; i += (long long)gridDim.x * blockDim.x) {
    long long v[3];
    node_ijk(i, L.Nn, v[0], v[1], v[2]);
    double acc = 0.0;
    for (int q = 0; q < 8; ++q) {
      long long c[3];
      double w = 1.0;
      bool use = true;
      for (int a = 0; a < 3; ++a) {
        const int bit = (q >> a) & 1;
        if (v[a] & 1) {
          c[a] = v[a] / 2 + bit;
          w *= 0.5;
        } else {
          use = use && !bit;
          c[a] = v[a] / 2;
        }
      }
      if (use) acc += w * (double)xc[(c[0] * Nc + c[1]) * Nc + c[2]];
    }
    xf[i] = (float)acc;
  }
}

// trilinear sample of a node grid at points in input order (the iso-value): clamped to the border cells
__global__ void __launch_bounds__(kThreads) grid_sample_kernel(const double* __restrict__ pts, long long n, Level L, const float* __restrict__ grid,
                                                               float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long c[3];
    double t[3];
    for (int a = 0; a < 3; ++a) {
      const double q = __ddiv_rn(__dsub_rn(pts[3 * i + a], L.o[a]), L.hw);
      const double f = floor(q);
      c[a] = f < 0.0 ? 0 : (f > (double)(L.R - 1) ? L.R - 1 : (long long)f);
      t[a] = __dsub_rn(q, (double)c[a]);
    }
    double acc = 0.0;
    for (int q = 0; q < 8; ++q) {
      const int bx = q & 1, by = (q >> 1) & 1, bz = (q >> 2) & 1;
      acc = __dadd_rn(acc, __dmul_rn(corner_phi(t, bx, by, bz), (double)grid[((c[0] + bx) * L.Nn + c[1] + by) * L.Nn + c[2] + bz]));
    }
    out[i] = (float)acc;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
// Caller-owned device scratch for n points at the finest depth d, carved in a fixed order (base == nullptr: sizes only).
struct PScratch : GridBuffers {
  double* t;         // [n,3]
  double* samples;   // [n]
  int* cell_map;     // [R^3]
  float* vfield;     // [M,3]
  float *b, *ssq, *diag, *r, *zr, *p, *ap;  // [M]
  double* partial;   // [3 * kRedBlocks]
  double* scalars;   // [2]: a, a / h^3
  Cg* cg;
  int* bad;
};

size_t pcarve(char* base, int n, int d, size_t cub_size, PScratch* s) {
  size_t off = 0;
  const size_t m = (size_t)n;
  const size_t R = (size_t)1 << d, M = (R + 1) * (R + 1) * (R + 1);
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
  s->flag = (int*)take(4 * m);
  s->cub = take(cub_size);
  s->cub_bytes = cub_size;
  s->t = (double*)take(24 * m);
  s->samples = (double*)take(8 * m);
  s->cell_map = (int*)take(4 * R * R * R);
  s->vfield = (float*)take(12 * M);
  s->b = (float*)take(4 * M);
  s->ssq = (float*)take(4 * M);
  s->diag = (float*)take(4 * M);
  s->r = (float*)take(4 * M);
  s->zr = (float*)take(4 * M);
  s->p = (float*)take(4 * M);
  s->ap = (float*)take(4 * M);
  s->partial = (double*)take(8 * 3 * kRedBlocks);
  s->scalars = (double*)take(16);
  s->cg = (Cg*)take(sizeof(Cg));
  s->bad = (int*)take(4);
  return off;
}

bool valid_size(int64_t n, int32_t depth) { return n >= 1 && n <= 2147483647LL && depth >= 2 && depth <= kMaxDepth; }

int bind_pscratch(const char* what, int n, int d, void* scratch, size_t scratch_bytes, PScratch* s) {
  size_t cb = 0;
  if (int rc = grid_cub_bytes(n, &cb)) return rc;
  const size_t need = pcarve(nullptr, n, d, cb, s);
  if (!scratch || scratch_bytes < need) {
    set_error("%s: scratch too small: need %zu bytes, got %zu", what, need, scratch ? scratch_bytes : (size_t)0);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  pcarve(static_cast<char*>(scratch), n, d, cb, s);
  return FNR_OK;
}

bool valid_cube(const double* origin, double side) {
  return origin && std::isfinite(origin[0]) && std::isfinite(origin[1]) && std::isfinite(origin[2]) && std::isfinite(side) && side > 0.0;
}

int grid_blocks(long long work) { return grid_for(work, kThreads, kRedBlocks); }

// Refuses non-finite points and points outside the cube (one host read).
int check_inside(const char* what, const double* points, int n, const Level& L, const PScratch& s, cudaStream_t st) {
  if (int rc = check_cuda(cudaMemsetAsync(s.bad, 0, sizeof(int), st), "cudaMemsetAsync")) return rc;
  poisson_check_kernel<<<grid_blocks(n), kThreads, 0, st>>>(points, n, L, s.bad);
  if (int rc = check_launch("poisson_check_kernel")) return rc;
  int bad = 0;
  if (int rc = check_cuda(cudaMemcpyAsync(&bad, s.bad, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync")) return rc;
  if (int rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize")) return rc;
  if (bad) {
    set_error("%s: a point is not finite or lies outside the cube", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  return FNR_OK;
}

// Sort at depth L.d, then the splat and the right-hand side into scratch (or the caller's outputs).
int sort_and_splat(const double* points, int n, const Level& L, const PScratch& s, KSplat A, float* vfield, float* b, cudaStream_t st, Sorted* out) {
  Grid g;
  if (int rc = build_grid(points, n, L.o, L.hw, s, st, &g)) return rc;
  const int nb = grid_for(n, kThreads, INT_MAX);
  frac_kernel<<<nb, kThreads, 0, st>>>(g, L, s.t);
  if (int rc = check_launch("frac_kernel")) return rc;
  fill_int_kernel<<<grid_blocks(L.R * L.R * L.R), kThreads, 0, st>>>(s.cell_map, L.R * L.R * L.R, -1);
  if (int rc = check_launch("fill_int_kernel")) return rc;
  cell_map_kernel<<<nb, kThreads, 0, st>>>(g, L, s.cell_map);
  if (int rc = check_launch("cell_map_kernel")) return rc;
  area_kernel<<<1, 1, 0, st>>>(s.ncells, n, L, s.scalars);
  if (int rc = check_launch("area_kernel")) return rc;
  const Sorted S{n, s.perm, s.keys, s.t, s.cstart, s.cell_map};
  A.scalars = s.scalars;
  A.vfield = vfield;
  A.ssq = s.ssq;
  splat_kernel<<<grid_blocks(L.M), kThreads, 0, st>>>(S, L, A);
  if (int rc = check_launch("splat_kernel")) return rc;
  rhs_kernel<<<grid_blocks(L.M), kThreads, 0, st>>>(L, vfield, b);
  if (int rc = check_launch("rhs_kernel")) return rc;
  *out = S;
  return FNR_OK;
}

int apply(const Sorted& S, const Level& L, const PScratch& s, double alpha, const float* x, float* y, double* partial, cudaStream_t st) {
  point_sample_kernel<<<grid_for(S.n, kThreads, INT_MAX), kThreads, 0, st>>>(S, L, x, s.samples);
  if (int rc = check_launch("point_sample_kernel")) return rc;
  apply_kernel<<<kRedBlocks, kThreads, 0, st>>>(S, L, s.scalars, alpha, x, s.samples, y, partial);
  return check_launch("apply_kernel");
}

int read_cg(const PScratch& s, Cg* host, cudaStream_t st) {
  if (int rc = check_cuda(cudaMemcpyAsync(host, s.cg, sizeof(Cg), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync")) return rc;
  return check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
}

// Preconditioned CG on one level from the initial guess in x; *iters and *rel (|r| / |b|) on return.
int cg_solve(const Sorted& S, const Level& L, const PScratch& s, double alpha, int max_iters, double tol, float* x, int64_t* iters, double* rel,
             cudaStream_t st) {
  diag_kernel<<<grid_blocks(L.M), kThreads, 0, st>>>(L, s.scalars, alpha, s.ssq, s.diag);
  if (int rc = check_launch("diag_kernel")) return rc;
  if (int rc = apply(S, L, s, alpha, x, s.ap, nullptr, st)) return rc;
  cg_init_kernel<<<kRedBlocks, kThreads, 0, st>>>(L.M, s.b, s.ap, s.diag, s.r, s.zr, s.p, s.partial);
  if (int rc = check_launch("cg_init_kernel")) return rc;
  cg_scalars_kernel<<<1, kThreads, 0, st>>>(s.partial, kCgInit, s.cg);
  if (int rc = check_launch("cg_scalars_kernel")) return rc;
  Cg h{};
  if (int rc = read_cg(s, &h, st)) return rc;
  const double bb = h.bb, stop = tol * tol * bb;
  int it = 0;
  while (bb > 0.0 && h.rr > stop && it < max_iters) {
    if (int rc = apply(S, L, s, alpha, s.p, s.ap, s.partial, st)) return rc;
    cg_scalars_kernel<<<1, kThreads, 0, st>>>(s.partial, kCgAlpha, s.cg);
    if (int rc = check_launch("cg_scalars_kernel")) return rc;
    cg_update_kernel<<<kRedBlocks, kThreads, 0, st>>>(L.M, s.cg, s.p, s.ap, s.diag, x, s.r, s.zr, s.partial);
    if (int rc = check_launch("cg_update_kernel")) return rc;
    cg_scalars_kernel<<<1, kThreads, 0, st>>>(s.partial, kCgBeta, s.cg);
    if (int rc = check_launch("cg_scalars_kernel")) return rc;
    ++it;
    if (int rc = read_cg(s, &h, st)) return rc;
    if (h.rr <= stop || it >= max_iters) break;
    cg_direction_kernel<<<grid_blocks(L.M), kThreads, 0, st>>>(L.M, s.cg, s.zr, s.p);
    if (int rc = check_launch("cg_direction_kernel")) return rc;
  }
  *iters = it;
  *rel = bb > 0.0 ? std::sqrt(h.rr / bb) : 0.0;
  return FNR_OK;
}

}  // namespace

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_poisson_scratch_bytes(int64_t num_points, int32_t depth, size_t* bytes) {
  if (!bytes || !valid_size(num_points, depth)) {
    set_error("invalid arguments to fnr_poisson_scratch_bytes (n = %lld, depth %d)", (long long)num_points, depth);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  size_t cb = 0;
  if (int rc = grid_cub_bytes((int)num_points, &cb)) return rc;
  PScratch s;
  *bytes = pcarve(nullptr, (int)num_points, depth, cb, &s);
  return FNR_OK;
}

int fnr_poisson_splat(const double* points, const float* normals, const float* colors, const float* fruit, int64_t num_points, int32_t depth,
                      const double* origin, double side, void* scratch, size_t scratch_bytes, float* density, float* normal_field,
                      float* node_colors, float* node_fruit, float* rhs, void* stream) {
  const char* what = "fnr_poisson_splat";
  if (!points || !normals || !valid_size(num_points, depth) || !valid_cube(origin, side) || !density || !normal_field || !rhs ||
      !colors != !node_colors || !fruit != !node_fruit) {
    set_error("invalid arguments to %s (n = %lld, depth %d, side %g)", what, (long long)num_points, depth, side);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const int n = (int)num_points;
  PScratch s;
  if (int rc = bind_pscratch(what, n, depth, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Level L = make_level(depth, origin, side);
  if (int rc = check_inside(what, points, n, L, s, st)) return rc;
  KSplat A{normals, colors, fruit, nullptr, density, nullptr, node_colors, node_fruit, nullptr};
  Sorted S;
  return sort_and_splat(points, n, L, s, A, normal_field, rhs, st, &S);
}

int fnr_poisson_apply(int64_t num_points, int32_t depth, float alpha, const void* scratch, size_t scratch_bytes, const float* x, float* y,
                      void* stream) {
  const char* what = "fnr_poisson_apply";
  if (!x || !y || !valid_size(num_points, depth) || !std::isfinite(alpha) || alpha < 0.f) {
    set_error("invalid arguments to %s (n = %lld, depth %d, alpha %g)", what, (long long)num_points, depth, (double)alpha);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  PScratch s;
  if (int rc = bind_pscratch(what, (int)num_points, depth, const_cast<void*>(scratch), scratch_bytes, &s)) return rc;
  const double zero[3] = {0.0, 0.0, 0.0};
  const Level L = make_level(depth, zero, 1.0);  // the operator does not depend on the cube's placement
  const Sorted S{(int)num_points, s.perm, s.keys, s.t, s.cstart, s.cell_map};
  return apply(S, L, s, (double)alpha, x, y, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_poisson_solve(const double* points, const float* normals, const float* colors, const float* fruit, int64_t num_points, int32_t depth,
                      const double* origin, double side, float alpha, int32_t max_iters, float tolerance, void* scratch, size_t scratch_bytes,
                      float* chi, float* density, float* node_colors, float* node_fruit, int64_t* iterations, double* residual, void* stream) {
  const char* what = "fnr_poisson_solve";
  if (!points || !normals || !valid_size(num_points, depth) || !valid_cube(origin, side) || !chi || !density || !iterations || !residual ||
      !colors != !node_colors || !fruit != !node_fruit || !std::isfinite(alpha) || alpha < 0.f || max_iters < 0 ||
      !std::isfinite(tolerance) || tolerance < 0.f) {
    set_error("invalid arguments to %s (n = %lld, depth %d, side %g, alpha %g, max_iters %d, tolerance %g)", what, (long long)num_points, depth,
              side, (double)alpha, max_iters, (double)tolerance);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const int n = (int)num_points;
  PScratch s;
  if (int rc = bind_pscratch(what, n, depth, scratch, scratch_bytes, &s)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (int rc = check_inside(what, points, n, make_level(depth, origin, side), s, st)) return rc;
  const int d0 = depth > 4 ? std::max(depth - 3, 4) : depth;
  iterations[0] = iterations[1] = 0;
  for (int d = d0; d <= depth; ++d) {
    const Level L = make_level(d, origin, side);
    const bool fine = d == depth;
    KSplat A{normals, colors, fruit, nullptr, fine ? density : nullptr, nullptr, fine ? node_colors : nullptr, fine ? node_fruit : nullptr, nullptr};
    Sorted S;
    if (int rc = sort_and_splat(points, n, L, s, A, s.vfield, s.b, st, &S)) return rc;
    if (d == d0) {
      if (int rc = check_cuda(cudaMemsetAsync(chi, 0, sizeof(float) * (size_t)L.M, st), "cudaMemsetAsync")) return rc;
    } else {
      prolong_kernel<<<grid_blocks(L.M), kThreads, 0, st>>>(L, chi, s.ap);
      if (int rc = check_launch("prolong_kernel")) return rc;
      if (int rc = check_cuda(cudaMemcpyAsync(chi, s.ap, sizeof(float) * (size_t)L.M, cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync")) return rc;
    }
    int64_t it = 0;
    if (int rc = cg_solve(S, L, s, (double)alpha, max_iters, (double)tolerance, chi, &it, residual, st)) return rc;
    iterations[1] += it;
    if (fine) iterations[0] = it;
  }
  return FNR_OK;
}

int fnr_poisson_sample(const double* points, int64_t num_points, int32_t depth, const double* origin, double side, const float* grid, float* out,
                       void* stream) {
  if (!points || !grid || !out || num_points < 1 || depth < 2 || depth > kMaxDepth || !valid_cube(origin, side)) {
    set_error("invalid arguments to fnr_poisson_sample (n = %lld, depth %d, side %g)", (long long)num_points, depth, side);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const Level L = make_level(depth, origin, side);
  grid_sample_kernel<<<grid_blocks(num_points), kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(points, num_points, L, grid, out);
  return check_launch("grid_sample_kernel");
}

}  // extern "C"
