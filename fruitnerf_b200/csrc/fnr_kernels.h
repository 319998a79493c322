// Internal kernel-argument structs and launcher prototypes (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fnr_common.cuh"

namespace fnr {

struct KField {
  int L, log2T, num_images;
  int position_mode, appearance_mode, pass_semantic_gradients;
  float scalings[FNR_MAX_LEVELS];
  float aabb[6];
};

struct KParams {
  float* hash_table;
  float* base_w[FNR_MAX_LAYERS];
  float* base_b[FNR_MAX_LAYERS];
  float* sem_w[FNR_MAX_LAYERS];
  float* sem_b[FNR_MAX_LAYERS];
  float* head_w;
  float* head_b;
  float* col_w[FNR_MAX_LAYERS];
  float* col_b[FNR_MAX_LAYERS];
  float* app_embedding;
};

struct KRays {
  int R, S;
  const float* origins;
  const float* directions;
  const float* starts;
  const float* ends;
  const int32_t* camera_indices;
};

struct KFieldOut {
  float* sample_density;
  float* sample_rgb;
  float* sample_semantics;
  float* stash_encoding;
};

struct KComposite {
  const float* sample_density;
  const float* sample_rgb;
  const float* sample_semantics;
  float* rgb;
  float* accumulation;
  float* depth;
  int32_t* depth_index;
  float* semantics;
  float* weights;
  int clamp_rgb;
};

struct KCompositeBwd {
  const float* weights;
  const float* sample_density;
  const float* sample_rgb;
  const float* sample_semantics;
  const float* accumulation;
  const float* d_rgb;
  const float* d_accumulation;
  const float* d_semantics;
  const float* d_weights;
  const float* d_sample_density;
  const float* d_sample_rgb;
  const float* d_sample_semantics;
  float* point_grads;  // [N,5]: d_density, d_rgb[3], d_logit
  int pass_semantic_gradients;
};

struct KFieldBwd {
  const float* point_grads;     // [N,5]
  const float* stash_encoding;  // [N,32] or NULL (recompute)
};

struct KExport {
  int B, S;
  const float* origins;  // [B,3]
  float normal[3];
  const float* bins;  // [S+1] spacing bins in [0,1], or [B,S+1] with bins_ray_stride = S+1 (per-ray jitter)
  int bins_ray_stride;
  float near_plane, far_plane;
  float logit_min, density_min, label_thr;
  int capacity;
  uint64_t point_base;
  float* rows[3];
  uint64_t* keys[3];
  int32_t* counts;
  float* sample_rgb;
  float* point_location;
  float* sample_semantics;
  float* sample_density;
  int64_t* semantics_colormap;
};

// ---- per-ray glue kernels (fnr_glue.cu) ----
struct KPixelBatch {
  int R, N, H, W;
  float fx, fy, cx, cy;
  const float* rand;     // [R,3] uniform draws
  const float* c2w;      // [N,3,4]
  const float* images;   // [N,H,W,3]
  const float* masks;    // [N,H,W,1]
  float* origins;        // [R,3]
  float* directions;     // [R,3]
  int32_t* camera_indices;  // [R]
  int64_t* indices;      // [R,3] (image, row, col) or NULL
  float* image;          // [R,3]
  float* fruit_mask;     // [R,1]
};
struct KSpacedBins {
  int R, S, mode;        // mode 0 = uniform, 1 = linear-in-disparity piecewise
  const float* base_bins;  // [S+1] linspace(0,1,S+1) made by the caller
  const float* t_rand;   // NULL | [R] (t_stride 1) | [R,S+1]
  int t_stride;
  const float* nears;    // [R]
  const float* fars;     // [R]
  float* bins;           // [R,S+1]
  float* starts;         // [R,S]
  float* ends;           // [R,S]
};
struct KLosses {
  int R;
  float semantic_weight;
  const float* rgb;        // [R,3]
  const float* semantics;  // [R]
  const float* image;      // [R,3]
  const float* fruit_mask; // [R]
  float* out;              // [4]: mse, weight*bce, psnr, -
  float* d_rgb;            // [R,3] d mse / d rgb (may be NULL)
  float* d_semantics;      // [R]   d (weight*bce) / d semantics (may be NULL)
};
struct KRayMetrics {
  int R, S;
  const float* weights;  // [R,S]
  const float* sdist;    // [R,S+1] (distortion only)
  const float* starts;   // [R,S]   (median depth only)
  const float* ends;
  float* distortion;     // scalar, pre-zeroed, or NULL
  float* depth;          // [R] or NULL
};
int launch_pixel_batch(const KPixelBatch& A, cudaStream_t st);
int launch_spaced_bins(const KSpacedBins& A, cudaStream_t st);
int launch_render_losses(const KLosses& A, cudaStream_t st);
int launch_ray_metrics(const KRayMetrics& A, cudaStream_t st);

// ---- optimiser (fnr_optim.cu) ----
constexpr int kMaxAdamTensors = 48;
struct KAdamTensor {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  long long n;
  int vec4;  // all four pointers 16-byte aligned
};
struct KAdam {
  int count;
  KAdamTensor t[kMaxAdamTensors];
};
int launch_adam(const KAdam& A, int radam, const float* hyper, cudaStream_t st);

// ---- proposal stage (fnr_proposal.cu) ----
struct KDensity {  // nerfstudio HashMLPDensityField: hash grid (L levels, F=2) -> Linear(2L,16) -> ReLU -> Linear(16,1)
  int L, log2T, position_mode;
  float scalings[FNR_MAX_LEVELS];
  float aabb[6];
  float* hash_table;
  float* w0;
  float* b0;
  float* w1;
  float* b1;
};

struct KPdf {
  int R, S, num_samples;
  const float* weights;        // [R,S]
  const float* existing_bins;  // [R,S+1] spacing bins of the previous level
  const float* u_base;         // [num_samples+1] = linspace(0, 1 - 1/NB, NB) made by the host
  const float* u_rand;         // NULL (bin centres) | [R*u_stride]
  int u_stride;                // 1 = single jitter per ray, num_samples+1 = per bin
  float anneal, hist_padding, eps;
  const float* anneal_dev;     // optional device scalar overriding `anneal` (CUDA-graph replays with a moving schedule)
  const float* nears;          // [R]
  const float* fars;           // [R]
  float* new_bins;             // [R,num_samples+1]
  float* starts;               // [R,num_samples]
  float* ends;                 // [R,num_samples]
};

struct KInterlevel {
  int R, Sc, Sp;
  const float* c;   // [R,Sc+1] final-level spacing bins
  const float* w;   // [R,Sc]   final-level weights
  const float* cp;  // [R,Sp+1] proposal spacing bins
  const float* wp;  // [R,Sp]   proposal weights
  float scale;      // mult / (R * Sc)
  float* loss;      // accumulated into (1 float)
  float* d_wp;      // [R,Sp] or NULL
};

int launch_proposal_weights_forward(const KDensity& D, const KRays& Rr, float* density, float* weights, cudaStream_t st);
int launch_proposal_weights_backward(const KDensity& D, const KDensity& G, const KRays& Rr, const float* density, const float* weights,
                                     const float* d_weights, cudaStream_t st);
int launch_pdf_sample(const KPdf& A, cudaStream_t st);
int launch_interlevel_loss(const KInterlevel& A, cudaStream_t st);
int proposal_limits(int* max_levels, int* hidden, int* max_bins);

int sm_count();

// Blocks for `work` items at `per_block` items per block: at least 1, at most `max_blocks`.
inline int grid_for(long long work, int per_block, int max_blocks) {
  long long b = (work + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

// Field kernels of fnr_simt.cu for a shipped family: tc selects the tensor-core (wgmma, sm_90a) instantiation, otherwise
// the exact-fp32 simt one.
int launch_field_forward(Family fam, bool tc, const KField& F, const KParams& P, const KRays& Rr, const KFieldOut& O, cudaStream_t st);
int launch_field_backward(Family fam, bool tc, const KField& F, const KParams& P, const KParams& G, const KRays& Rr, const KFieldBwd& B,
                          cudaStream_t st);
int launch_export(Family fam, bool tc, const KField& F, const KParams& P, const KExport& E, cudaStream_t st);
int launch_simt_composite(const KRays& Rr, const KComposite& Cm, cudaStream_t st);
int launch_simt_composite_backward(const KRays& Rr, const KCompositeBwd& B, cudaStream_t st);
int launch_hash_indices(const KField& F, const KRays& Rr, int32_t* rows, float* positions, cudaStream_t st);

}  // namespace fnr
