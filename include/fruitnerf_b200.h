/*
 * fruitnerf_b200 -- C ABI of the H100-native FruitNeRF hot path.
 *
 * One shared library (libfruitnerf_b200.so, sm_90a) behind the reference's Nerfstudio plugin
 * surface.  Plain C: no C++ or torch types cross this boundary.  Every buffer is a raw DEVICE
 * pointer allocated and owned by the caller (PyTorch on the Python side); the library keeps no
 * global state besides a thread-local error string and, once the fruit_nerf_big backward has run, a cuBLAS
 * handle (resolved with dlopen; used for that family's weight-gradient GEMMs only).  All kernels are enqueued on the
 * `cudaStream_t` passed as `void* stream` and never synchronise the host.
 *
 * Return value of every entry point: 0 = OK, negative = error (see FNR_ERR_*); the message is
 * available from fnr_last_error().  No exceptions, no exit().
 *
 * Reference interfaces replaced (file:line under /root/reference):
 *   fnr_render_forward   FruitModel.get_outputs after the sampler: FruitField.forward +
 *                        RaySamples.get_weights + RGB/Depth/Accumulation/Semantic renderers
 *                        (fruit_nerf/fruit_nerf.py:320-348; fruit_nerf/fruit_field.py:168-301)
 *   fnr_render_backward  autograd of the above (the reference gets it from torch/tcnn autograd;
 *                        loss inputs of fruit_nerf/fruit_nerf.py:359-366)
 *                        -- with only the sample_* outputs requested (ray-level pointers NULL)
 *                        this is FruitField.forward alone (fruit_nerf/fruit_field.py:283-301)
 *   fnr_export_forward   FruitModel.get_export_outputs + the threshold/selection loop body of
 *                        sample_volume (fruit_nerf/fruit_nerf.py:251-269;
 *                        fruit_nerf/export/exporter_utils.py:100-153;
 *                        fruit_nerf/components/ray_samplers.py:54-104)
 *   fnr_proposal_weights_forward/backward, fnr_pdf_sample, fnr_interlevel_loss
 *                        the proposal stage FruitModel builds from nerfstudio parts
 *                        (fruit_nerf/fruit_nerf.py:149-206 construction, :320-321 call, :361-364
 *                        interlevel loss): HashMLPDensityField.get_density + get_weights,
 *                        PDFSampler.generate_ray_samples, nerfstudio losses.interlevel_loss
 *   fnr_pixel_batch, fnr_spaced_bins, fnr_render_losses, fnr_ray_metrics
 *                        the per-ray glue of a training iteration: pixel sampling + ray generation
 *                        (fruit_nerf/data/fruit_datamanager.py:183-192), the initial spaced sampler
 *                        (components/ray_samplers.py:54-104), losses and metrics (fruit_nerf.py:359-366, 396-401),
 *                        proposal-level median depths (fruit_nerf.py:339-340)
 *   fnr_adam_step        torch.optim.Adam / RAdam over a param group (nerfstudio Optimizers; optimiser
 *                        settings fruit_nerf/fruit_nerf_config.py:47-56, 90-103, 140-153)
 *   fnr_radius_count, fnr_voxel_down_sample, fnr_dbscan, fnr_cluster_sums
 *                        stages 1-2 of the fruit counting (clustering/clustering_base.py:138-143, 183-259):
 *                        radius-outlier removal, voxel down-sampling, DBSCAN, the sums of the centre merge
 *   fnr_backproject_select, fnr_knn_mean_distance, fnr_estimate_normals
 *                        the `pointcloud` export (fruit_nerf/scripts/exporter.py:124-129, nerfstudio ExportPointCloud):
 *                        back-projection and selection of rendered rays, statistical outlier removal, normal estimation
 *   fnr_icp_scaled, fnr_ward_cut, fnr_hausdorff
 *                        stage 3 of the fruit counting (clustering/clustering_base.py:261-429): scaled ICP of the fruit
 *                        template, Ward sub-centres for k = 2..6 and Hausdorff distances of each group to split
 */
#ifndef FRUITNERF_B200_H
#define FRUITNERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FNR_ABI_VERSION 2
#define FNR_MAX_LEVELS 32
#define FNR_MAX_LAYERS 4
#define FNR_MAX_WIDTH 128

#define FNR_OK 0
#define FNR_ERR_INVALID_ARGUMENT (-1)
#define FNR_ERR_UNSUPPORTED (-2)
#define FNR_ERR_CUDA (-3)

/* position_mode: how FruitField.get_density maps world positions to [0,1]^3
 * (fruit_nerf/fruit_field.py:170-175). */
#define FNR_POS_CONTRACT 0 /* (SceneContraction_inf(x) + 2) / 4  -- training / inference */
#define FNR_POS_AABB 1     /* (x - aabb_min) / (aabb_max - aabb_min) -- export, after setup_inference */

/* appearance_mode: which appearance embedding feeds the colour MLP
 * (fruit_nerf/fruit_field.py:250-260, 217-219). */
#define FNR_APP_PER_CAMERA 0 /* embedding[camera_index]  (self.training) */
#define FNR_APP_MEAN 1       /* embedding.mean(0)        (inference/export, or use_average...) */
#define FNR_APP_ZEROS 2      /* zeros                    (eval without average embedding) */

/* implementation selector for the forward, export and backward kernels */
#define FNR_IMPL_AUTO 0    /* tensor-core kernels (every shape that passes validation has them) */
#define FNR_IMPL_SIMT 1    /* fp32 CUDA-core kernels (exact-fp32 device reference) */
#define FNR_IMPL_TCGEN05 2 /* tensor-core kernels, as AUTO (wgmma on sm_90a; historical name) */

/* One nn.Linear stack: n_layers Linear layers, ReLU between them (nerfstudio MLP torch path);
 * dims[0] = input width, dims[n_layers] = output width. */
typedef struct fnr_mlp_desc {
  int32_t n_layers;
  int32_t dims[FNR_MAX_LAYERS + 1];
} fnr_mlp_desc;

/* Static description of a FruitField (fruit_nerf/fruit_field.py:70-166). */
typedef struct fnr_field_desc {
  int32_t num_levels;                /* L */
  int32_t features_per_level;        /* F, must be 2 */
  int32_t log2_hashmap_size;         /* T */
  float scalings[FNR_MAX_LEVELS];    /* per-level scale, taken from the host module as is */
  int32_t geo_feat_dim;              /* 15 / 30 */
  int32_t appearance_dim;            /* 32 */
  int32_t num_images;                /* rows of the appearance embedding */
  fnr_mlp_desc base;                 /* L*F -> hidden -> 1+geo */
  fnr_mlp_desc semantic;             /* geo -> ... -> sem_out (no output activation) */
  fnr_mlp_desc color;                /* 16+geo+app -> ... -> 3, sigmoid */
  float aabb[6];                     /* min xyz, max xyz (FNR_POS_AABB) */
  int32_t position_mode;             /* FNR_POS_* */
  int32_t appearance_mode;           /* FNR_APP_* */
  int32_t pass_semantic_gradients;   /* 0: semantic MLP sees detach(geo), semantics use detach(w) */
  int32_t impl;                      /* FNR_IMPL_* */
} fnr_field_desc;

/* fp32 device pointers in torch layouts (Linear weight = [out][in] row-major).  The same struct
 * describes the gradient buffers for fnr_render_backward (all fields then writable, accumulated
 * into with atomics: the caller zero-fills or pre-loads them). */
typedef struct fnr_field_params {
  float* hash_table;                 /* [L * 2^T, F] */
  float* base_w[FNR_MAX_LAYERS];
  float* base_b[FNR_MAX_LAYERS];
  float* sem_w[FNR_MAX_LAYERS];
  float* sem_b[FNR_MAX_LAYERS];
  float* head_w;                     /* SemanticFieldHead Linear: [1][sem_out] */
  float* head_b;                     /* [1] */
  float* col_w[FNR_MAX_LAYERS];
  float* col_b[FNR_MAX_LAYERS];
  float* app_embedding;              /* [num_images][appearance_dim] */
} fnr_field_params;

/* A batch of R rays with S samples each (nerfstudio RaySamples after the sampler). */
typedef struct fnr_ray_batch {
  int32_t num_rays;                  /* R */
  int32_t num_samples;               /* S */
  const float* origins;              /* [R,3] */
  const float* directions;           /* [R,3] */
  const float* starts;               /* [R,S] frustum starts */
  const float* ends;                 /* [R,S] frustum ends   */
  const int32_t* camera_indices;     /* [R] or NULL (required for FNR_APP_PER_CAMERA) */
} fnr_ray_batch;

/* Outputs of the render forward.  Any pointer may be NULL to skip that output. */
typedef struct fnr_render_out {
  float* rgb;                        /* [R,3]  sum(w*c) + c_last*(1-sum w) */
  float* accumulation;               /* [R]    sum w */
  float* depth;                      /* [R]    median depth */
  int32_t* depth_index;              /* [R]    median sample index (searchsorted left, clamped) */
  float* semantics;                  /* [R]    sum(w * logit) */
  float* weights;                    /* [R,S] */
  float* sample_density;             /* [R,S]   field outputs per sample ... */
  float* sample_rgb;                 /* [R,S,3] */
  float* sample_semantics;           /* [R,S]   (logit) */
  float* stash_encoding;             /* [R,S,L*F] encoded features kept for the backward (32-byte aligned), or NULL */
  int32_t clamp_rgb;                 /* 1: eval-mode RGBRenderer (nan_to_num + clamp to [0,1]) */
} fnr_render_out;

/* Gradients flowing into the render backward.  NULL = zero. */
typedef struct fnr_render_grads {
  const float* d_rgb;                /* [R,3] */
  const float* d_accumulation;       /* [R]   */
  const float* d_semantics;          /* [R]   */
  const float* d_weights;            /* [R,S] */
  const float* d_sample_density;     /* [R,S]   direct per-sample grads (FruitField.forward users) */
  const float* d_sample_rgb;         /* [R,S,3] */
  const float* d_sample_semantics;   /* [R,S]   */
} fnr_render_grads;

/* Forward products the backward re-reads (written by fnr_render_forward). */
typedef struct fnr_render_saved {
  const float* weights;              /* [R,S] */
  const float* sample_density;       /* [R,S] */
  const float* sample_rgb;           /* [R,S,3] */
  const float* sample_semantics;     /* [R,S] */
  const float* stash_encoding;       /* [R,S,L*F] */
  const float* accumulation;         /* [R] */
} fnr_render_saved;

/* Export: thresholds and compacted outputs of sample_volume's loop body
 * (fruit_nerf/export/exporter_utils.py:111-153). */
typedef struct fnr_export_params {
  float semantic_logit_min;          /* 3.0   : mask_sem  = logit   >= 3    */
  float density_min;                 /* 70.0  : mask_den  = density >= 70   */
  float label_sigmoid_threshold;     /* 0.9   : label = heaviside(sigmoid(logit) - 0.9) */
  int32_t capacity;                  /* rows available in each of the three output sets */
  int32_t bins_ray_stride;           /* 0: one bins[S+1] array shared by every ray (deterministic grid); S+1: per-ray
                                      * bins[B,S+1] -- the stratified jitter UniformSamplerWithNoise applies while its
                                      * module is in training mode (components/ray_samplers.py:78-87), which is the state
                                      * the reference exporter runs it in (a module created after eval_setup()) */
} fnr_export_params;

typedef struct fnr_export_out {
  /* set 0: label & density ("semantic_colormap"), set 1: logit & density ("semantic"),
   * set 2: density only ("density").  Each row: x y z r g b a, a = sigmoid(logit) for sets 0/1
   * and sigmoid(density) for set 2.  counts[3] are device counters the caller zeroes before the
   * first batch; rows beyond capacity are counted but not written. */
  float* rows[3];                    /* [capacity,7] each */
  uint64_t* keys[3];                 /* [capacity] global point index (ray*S+sample) of each row, or NULL */
  int32_t* counts;                   /* [3] */
  /* optional dense per-point outputs (get_export_outputs), NULL to skip */
  float* sample_rgb;                 /* [B,S,3] */
  float* point_location;             /* [B,S,3] */
  float* sample_semantics;           /* [B,S] */
  float* sample_density;             /* [B,S] */
  int64_t* semantics_colormap;       /* [B,S] label in {0,1} */
} fnr_export_out;

/* ---- proposal-sampling stage (nerfstudio ProposalNetworkSampler as FruitModel builds it,
 * fruit_nerf/fruit_nerf.py:104-158, 318) ---- */

/* HashMLPDensityField: hash grid (num_levels, F=2, 2^log2_hashmap_size rows per level) ->
 * Linear(2*num_levels, 16) -> ReLU -> Linear(16, 1) -> trunc_exp * selector. */
typedef struct fnr_density_desc {
  int32_t num_levels;                /* <= 8 */
  int32_t log2_hashmap_size;
  int32_t hidden_dim;                /* 16 (proposal_net_args_list of all shipped configs) */
  float scalings[FNR_MAX_LEVELS];
  float aabb[6];
  int32_t position_mode;             /* FNR_POS_* */
} fnr_density_desc;

typedef struct fnr_density_params {  /* fp32 device pointers, torch layouts; also used for gradients */
  float* hash_table;                 /* [num_levels * 2^T, 2] */
  float* w0;                         /* [16][2*num_levels] */
  float* b0;                         /* [16] */
  float* w1;                         /* [1][16] */
  float* b1;                         /* [1] */
} fnr_density_params;

/* density_fn(frustum midpoints) + RaySamples.get_weights, fused: density [R,S] (may be NULL), weights [R,S]. */
int fnr_proposal_weights_forward(const fnr_density_desc* desc, const fnr_density_params* params, const fnr_ray_batch* rays,
                                 float* density, float* weights, void* stream);
/* d_weights [R,S] -> gradients of the proposal network (accumulated into `grads`). */
int fnr_proposal_weights_backward(const fnr_density_desc* desc, const fnr_density_params* params, const fnr_ray_batch* rays,
                                  const float* density, const float* weights, const float* d_weights,
                                  const fnr_density_params* grads, void* stream);

/* PDFSampler.generate_ray_samples (include_original = False) followed by the piecewise
 * linear-in-disparity spacing -> euclidean map of UniformLinDispPiecewiseSampler.
 *   weights [R,S], existing_bins [R,S+1] (spacing space), u_base [num_samples+1] = linspace(0, 1-1/NB, NB)
 *   (made by the caller, as the reference does with torch.linspace), u_rand NULL (bin centres, eval) or
 *   [R*u_stride] uniform draws (u_stride 1 = single jitter, num_samples+1 = per bin), weights are raised to
 *   `anneal` first (`anneal_dev`, when non-NULL, is a device scalar that overrides it: the annealing schedule
 *   can then advance between replays of a captured CUDA graph).  Outputs: new_bins [R,num_samples+1] (spacing), starts/ends [R,num_samples] (euclidean). */
int fnr_pdf_sample(const float* weights, const float* existing_bins, int32_t num_rays, int32_t num_existing,
                   int32_t num_samples, const float* u_base, const float* u_rand, int32_t u_stride, float anneal,
                   const float* anneal_dev, float histogram_padding, const float* nears, const float* fars,
                   float* new_bins, float* starts, float* ends, void* stream);

/* losses.interlevel_loss for ONE proposal level: adds mult * mean(lossfun_outer(c, w, cp, wp)) to *loss and
 * writes d loss / d wp into d_wp [R,Sp] (may be NULL).  c [R,Sc+1], w [R,Sc] are the (detached) final level. */
int fnr_interlevel_loss(const float* c, const float* w, const float* cp, const float* wp, int32_t num_rays, int32_t sc,
                        int32_t sp, float mult, float* loss, float* d_wp, void* stream);

/* One tensor of an optimiser param group: parameter, its gradient and the two Adam moments (all fp32, n elements). */
typedef struct fnr_adam_tensor {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t n;
} fnr_adam_tensor;

#define FNR_OPT_ADAM 0
#define FNR_OPT_RADAM 1
#define FNR_MAX_ADAM_TENSORS 48

/* torch.optim.Adam / RAdam step (amsgrad off, weight decay 0 -- the optimisers of
 * fruit_nerf/fruit_nerf_config.py:47-56, 90-103) for `count` tensors in ONE launch.  `tensors` is a HOST array;
 * `hyper` is a DEVICE array of 8 floats {lr, beta1, beta2, eps, 1-beta1^t, 1-beta2^t, radam_rect (<0: not
 * rectified), grad_scale}: the schedule advances by rewriting it, so the launch can live in a CUDA graph. */
int fnr_adam_step(const fnr_adam_tensor* tensors, int32_t count, int32_t kind, const float* hyper, void* stream);

/* ---- per-ray glue of a training iteration (fnr_glue.cu) ---------------------------------------------------- */

/* PixelSampler.sample + RayGenerator for a pinhole camera set held in device memory
 * (fruit_nerf/data/fruit_datamanager.py:183-192): rand [R,3] uniform draws -> (image, row, col) = floor(rand*[N,H,W]);
 * origins / directions [R,3] (pixel centres, normalised, OpenGL c2w [N,3,4]), camera_indices [R] int32,
 * indices [R,3] int64 (may be NULL), image [R,3] and fruit_mask [R,1] gathered from images [N,H,W,3] / masks [N,H,W,1]. */
int fnr_pixel_batch(const float* rand, const float* c2w, const float* images, const float* masks, int32_t num_images,
                    int32_t height, int32_t width, float fx, float fy, float cx, float cy, int32_t num_rays, float* origins,
                    float* directions, int32_t* camera_indices, int64_t* indices, float* image, float* fruit_mask,
                    void* stream);

#define FNR_SPACING_UNIFORM 0
#define FNR_SPACING_LINDISP_PIECEWISE 1
/* SpacedSampler.generate_ray_samples (components/ray_samplers.py:54-104; nerfstudio UniformLinDispPiecewiseSampler):
 * base_bins [S+1] = linspace(0,1,S+1) made by the caller; t_rand NULL (eval) | [R] (t_stride 1, single jitter) |
 * [R,S+1]; outputs spacing bins [R,S+1] and euclidean starts / ends [R,S]. */
int fnr_spaced_bins(const float* base_bins, const float* t_rand, int32_t t_stride, const float* nears, const float* fars,
                    int32_t num_rays, int32_t num_samples, int32_t mode, float* bins, float* starts, float* ends,
                    void* stream);

/* MSELoss(image, rgb), semantic_weight * BCEWithLogitsLoss(semantics, fruit_mask), PSNR (fruit_nerf.py:359-366,
 * 396-399) in one launch: out[0..2] = {mse, weighted bce, psnr}; d_rgb [R,3] / d_semantics [R] receive the gradients
 * of out[0] / out[1] (either may be NULL). */
int fnr_render_losses(const float* rgb, const float* semantics, const float* image, const float* fruit_mask,
                      int32_t num_rays, float semantic_weight, float* out, float* d_rgb, float* d_semantics,
                      void* stream);

/* nerfstudio distortion_loss of one level (mean over rays, ADDED to *distortion -- zero it first; fruit_nerf.py:400)
 * and / or DepthRenderer(method="median") of a level (fruit_nerf.py:339-340).  Pass NULL for the part not wanted. */
int fnr_ray_metrics(const float* weights, const float* sdist, const float* starts, const float* ends, int32_t num_rays,
                    int32_t num_samples, float* distortion, float* median_depth, void* stream);

int fnr_version(void);

/* Number of CUDA kernels this library has launched (or recorded into a stream capture) in this process since the
 * last call with reset != 0.  Diagnostic only: lets a benchmark report how many of ITS kernels a step consists of. */
uint64_t fnr_launch_count(int32_t reset);
const char* fnr_last_error(void);

/* FruitModel.get_outputs minus the sampler: field + compositing, fused. */
int fnr_render_forward(const fnr_field_desc* desc, const fnr_field_params* params, const fnr_ray_batch* rays,
                       const fnr_render_out* out, void* stream);

/* Gradients of fnr_render_forward w.r.t. every field parameter, accumulated into `grads`. */
int fnr_render_backward(const fnr_field_desc* desc, const fnr_field_params* params, const fnr_ray_batch* rays,
                        const fnr_render_saved* saved, const fnr_render_grads* upstream,
                        const fnr_field_params* grads, void* scratch, size_t scratch_bytes, void* stream);

/* Bytes of caller-allocated device scratch fnr_render_backward needs for this shape. */
int fnr_render_backward_scratch_bytes(const fnr_field_desc* desc, int32_t num_rays, int32_t num_samples, size_t* bytes);

/* Uniform-volume export of one ray batch: rays are `origins[b] + t * normal` (normal = 3 HOST
 * floats), sample s spans t in [bins[s], bins[s+1]] * far + (1 - bins) * near where `bins` is a
 * DEVICE array of S+1 spacing bins in [0,1] (the reference builds it with torch.linspace on the
 * host, components/ray_samplers.py:75; the caller does the same so the bits agree), or of
 * [num_rays, S+1] per-ray jittered bins when xp->bins_ray_stride = S+1.  The field
 * runs in FNR_POS_AABB / FNR_APP_MEAN mode.  `point_base` is the global index of this batch's
 * first point (for `keys`). */
int fnr_export_forward(const fnr_field_desc* desc, const fnr_field_params* params, const float* origins,
                       const float* normal, const float* bins, float near_plane, float far_plane,
                       int32_t num_rays, int32_t num_samples, uint64_t point_base,
                       const fnr_export_params* xp, const fnr_export_out* out, void* stream);

/* ---- gradient exchange of the data-parallel path (fruit_nerf/fruit_pipeline.py:116-118: DDP's all-reduce) as one kernel over
 * NVSwitch multicast memory.  The caller owns a SYMMETRIC allocation (every rank maps its own copy and the multicast object
 * spanning all copies; with PyTorch: torch.distributed._symmetric_memory.empty + rendezvous) and passes its addresses. ---- */
typedef struct fnr_nvls_desc {
  void* multicast_ptr;               /* multicast address of the fp32 gradient region */
  void* local_ptr;                   /* this rank's own (unicast) address of the same region */
  void* multicast_bf16;              /* bf16 staging region (numel bf16 elements) for wire_bf16, or NULL */
  void* local_bf16;
  void* const* signal_pads;          /* DEVICE array [world_size]: uint32 signal pad of every rank, zero-initialised */
  void* grid_counter;                /* device uint32, zero before the first call (wire_bf16 only), or NULL */
  int32_t rank, world_size;
  int32_t signal_slots;              /* uint32 slots in each pad */
  int32_t signal_slot_base;          /* first slot this library may use (up to 144 blocks x world_size slots from there) */
} fnr_nvls_desc;

/* In place: region[i] = mean over ranks of region[i], i < numel (numel % (8 * world_size) == 0).  Every rank calls it with
 * the same numel; the kernels of all ranks meet on the signal pads, so all ranks must launch it (like a collective).
 * wire_bf16 != 0: operands cross the links as bf16 (fp32 accumulation in the switch), result rounded to bf16. */
int fnr_nvls_allreduce_mean(const fnr_nvls_desc* d, size_t numel, int32_t wire_bf16, void* stream);

/* ---- fruit counting on the exported cloud: stages 1-2 of the reference clustering
 * (clustering/clustering_base.py:138-143 radius-outlier removal + voxel down-sampling, :183-207 DBSCAN, :209-259 the
 * cluster sums the centre merge runs on).  points: DEVICE [n,3] fp64, 0 <= n <= 2^31 - 1.  lo / hi: HOST arrays of 3
 * doubles, the per-axis minimum and maximum of the points (the grid origin and extent).  They must enclose every point:
 * with bounds that do not, points are clamped into the edge cells and counts, voxels and labels are undefined (no
 * out-of-bounds access; the calls do not detect it).  voxel_down_sample additionally needs lo to be the exact minimum,
 * as its keys are floor((p - lo) / voxel).  Every call needs the
 * caller-owned device scratch of fnr_cluster_scratch_bytes(n).  Distances are fp64, d2 = (dx*dx + dy*dy) + dz*dz with
 * no FMA, compared with <= r*r: scikit-learn's KD-tree radius_neighbors predicate.  Grid cells are keyed with 21 bits
 * per axis; a radius (eps, voxel size) that needs more cells on an axis returns FNR_ERR_UNSUPPORTED. ---- */

/* Bytes of device scratch any fruit-counting call on n points needs. */
int fnr_cluster_scratch_bytes(int64_t num_points, size_t* bytes);

/* counts[i] = min(cap, #{j : |p_i - p_j| <= radius}), the point itself included (cap >= 1): the neighbour counts of
 * radius-outlier removal (keep count - 1 >= nb_points, clustering_base.py:138-143) and of the DBSCAN core test. */
int fnr_radius_count(const double* points, int64_t num_points, const double* lo, const double* hi, double radius, int32_t cap,
                     int32_t* counts, void* scratch, size_t scratch_bytes, void* stream);

/* open3d voxel_down_sample as clustering.voxel_down_sample (clustering_base.py:141-143), bit for bit: voxel key
 * floor((p - lo) / voxel), one row per occupied voxel in lexicographic key order, the mean of its points summed in input
 * order.  out: DEVICE [n,3] (rows beyond *num_out untouched); *num_out: DEVICE int32. */
int fnr_voxel_down_sample(const double* points, int64_t num_points, const double* lo, const double* hi, double voxel, double* out,
                          int32_t* num_out, void* scratch, size_t scratch_bytes, void* stream);

/* sklearn.cluster.DBSCAN(eps, min_samples).labels_ (clustering_base.py:183-207): clusters are the connected components of
 * the core points (>= min_samples points within eps, itself included), numbered in increasing order of their smallest
 * core index; a non-core point within eps of a core takes the smallest such cluster label, any other point -1.
 * labels: DEVICE [n] int32; *num_clusters: DEVICE int32. */
int fnr_dbscan(const double* points, int64_t num_points, const double* lo, const double* hi, double eps, int32_t min_samples,
               int32_t* labels, int32_t* num_clusters, void* scratch, size_t scratch_bytes, void* stream);

/* Per-cluster fp64 coordinate sums [num_clusters,3] and point counts [num_clusters] of labels in [0, num_clusters) -- the
 * inputs of the centre merge (clustering_base.py:209-259).  Deterministic: the same input gives the same bits. */
int fnr_cluster_sums(const double* points, const int32_t* labels, int64_t num_points, int32_t num_clusters, double* sums,
                     int32_t* counts, void* scratch, size_t scratch_bytes, void* stream);

/* ---- the RGB surface cloud export (nerfstudio ExportPointCloud / generate_point_cloud as the reference CLI's
 * `pointcloud` subcommand runs it, fruit_nerf/scripts/exporter.py:124-129).  The k-nearest-neighbour calls take points,
 * bounds and scratch as the fruit-counting calls above (fnr_cluster_scratch_bytes(n)).  Neighbours are exact: the
 * min(k, n) points with the smallest fp64 distance, self included, ordered by (distance, input index).
 * 1 <= k <= 32; a larger k returns FNR_ERR_UNSUPPORTED. ---- */

/* mean_dist[i] = (sum of the Euclidean distances to the min(k, n) nearest neighbours of point i, added in ascending
 * order) / min(k, n): the per-point statistic of open3d remove_statistical_outlier.  mean_dist: DEVICE [n] fp64. */
int fnr_knn_mean_distance(const double* points, int64_t num_points, const double* lo, const double* hi, int32_t k, double* mean_dist,
                          void* scratch, size_t scratch_bytes, void* stream);

/* open3d estimate_normals with KNN(k): the unit eigenvector of the smallest eigenvalue of the (two-pass, fp64) covariance of
 * the min(k, n) nearest neighbours; (0, 0, 1) with fewer than 3 neighbours or a zero covariance.  The sign is the solver's.
 * view_dirs: DEVICE [n,3] fp32 or NULL; when given, a normal whose fp32 dot product with view_dirs[i] is > 0 is flipped.
 * normals: DEVICE [n,3] fp64. */
int fnr_estimate_normals(const double* points, int64_t num_points, const double* lo, const double* hi, int32_t k, const float* view_dirs,
                         double* normals, void* scratch, size_t scratch_bytes, void* stream);

/* One rendered batch of generate_point_cloud: point = origin + direction * depth in fp32 (multiply, then add), kept when
 * accumulation > 0.5 and, with use_bounding_box, box_min < point < box_max on every axis (box_min / box_max: HOST float[3]).
 * Kept rays are appended in ray order at row *count of points / colors (rgb) / view_dirs (direction), all DEVICE [capacity,3]
 * fp32; *count (DEVICE int32) is advanced by the number kept.  Rows at or beyond capacity are counted but not written.
 * origins, directions, rgb: DEVICE [R,3]; depth, accumulation: DEVICE [R]; all fp32. */
int fnr_backproject_select(const float* origins, const float* directions, const float* depth, const float* rgb, const float* accumulation,
                           int32_t num_rays, int32_t use_bounding_box, const float* box_min, const float* box_max, int32_t capacity,
                           float* points, float* colors, float* view_dirs, int32_t* count, void* stream);

/* ---- stage 3 of the fruit counting: the split of merged groups larger than one fruit (clustering_base.py:261-429).
 * Batched: one CTA per problem, fp64, distances (dx*dx + dy*dy) + dz*dz without FMA.  Segment bounds are DEVICE int64;
 * every other array is DEVICE fp64 unless stated.  Deterministic: the same input gives the same bits. */

/* open3d registration_icp(source, target_b, max_distance, translation(init_translation[b]),
 * TransformationEstimationPointToPoint(with_scaling=True), ICPConvergenceCriteria(relative_fitness, relative_rmse,
 * max_iteration)) for B targets that share one source: each iteration pairs every transformed source point with its
 * nearest target (lowest index on ties) when the squared distance is < max_distance^2, solves Umeyama with scale on the
 * pairs (identity with fewer than 3 pairs, zero spread or a cross-covariance of rank < 2) and left-multiplies it onto
 * the transform, until |d fitness| < relative_fitness and |d rmse| < relative_rmse.  source: [num_source,3]
 * (1..16384 points); target b: rows target_offsets[b] .. target_offsets[b+1] of targets, 1..max_targets <= 4096 rows
 * (a segment outside that range gets a NaN transform and iteration count -1).  Outputs: transforms [B,4,4] row-major,
 * fitness [B], rmse [B], iterations [B] int32 (updates applied). */
int fnr_icp_scaled(const double* source, int32_t num_source, const double* targets, const int64_t* target_offsets, int32_t num_problems,
                   int32_t max_targets, const double* init_translation, double max_distance, int32_t max_iteration,
                   double relative_fitness, double relative_rmse, double* transforms, double* fitness, double* rmse, int32_t* iterations,
                   void* stream);

/* sklearn AgglomerativeClustering(n_clusters=k, linkage="ward") sub-centres for k = 2..6 from one Ward tree per segment
 * (nearest-neighbour chain; ties go to the chain's predecessor, then to the lower cluster slot, a cluster's slot being
 * its smallest point index).  Segment b: rows offsets[b] .. offsets[b+1] of points, 1..max_points <= 4096 rows.
 * centres: [B,20,3]; rows 0-1 hold k = 2, 2-4 k = 3, 5-8 k = 4, 9-13 k = 5, 14-19 k = 6, each cut's sub-cluster means
 * ordered by smallest point index.  Rows of a cut with more clusters than points, and every row of a segment outside
 * 1..max_points, are NaN. */
int fnr_ward_cut(const double* points, const int64_t* offsets, int32_t num_segments, int32_t max_points, double* centres, void* stream);

/* Symmetric Hausdorff distance max(h(A_p, B_p), h(B_p, A_p)), exact, for num_pairs pairs: A_p is rows
 * a_ranges[2p] .. a_ranges[2p+1] of a, B_p rows b_ranges[2p] .. b_ranges[2p+1] of b.  distances: [num_pairs]; NaN for a
 * pair with an empty set. */
int fnr_hausdorff(const double* a, const int64_t* a_ranges, const double* b, const int64_t* b_ranges, int32_t num_pairs, double* distances,
                  void* stream);

/* Hash-grid row indices (exact-integer parity hook): rows[N,L,8] in nerfstudio corner order for
 * the masked [0,1]^3 positions of the given samples; also writes positions[N,3] if non-NULL. */
int fnr_hash_indices(const fnr_field_desc* desc, const fnr_ray_batch* rays, int32_t* rows, float* positions,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FRUITNERF_B200_H */
