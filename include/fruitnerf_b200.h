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
 *   fnr_radius_count_multi
 *                        radius counts for several radii on one grid: the parameter sweeps of
 *                        clustering/run_clustering_sweep.py
 *   fnr_backproject_select, fnr_knn_mean_distance, fnr_estimate_normals
 *                        the `pointcloud` export (fruit_nerf/scripts/exporter.py:124-129, nerfstudio ExportPointCloud):
 *                        back-projection and selection of rendered rays, statistical outlier removal, normal estimation
 *   fnr_icp_scaled, fnr_ward_cut, fnr_hausdorff
 *                        stage 3 of the fruit counting (clustering/clustering_base.py:261-429): scaled ICP of the fruit
 *                        template, Ward sub-centres for k = 2..6 and Hausdorff distances of each group to split
 *   fnr_camera_rays, fnr_compose_frame
 *                        the `render` command (debug/render.py, nerfstudio ns-render): camera-path rays and the
 *                        per-frame colour-mapped uint8 image
 *   fnr_pixel_batch_lens, fnr_camera_rays_lens
 *                        training and evaluation rays of captured data sets (fruit_nerf/data/fruitnerf_dataparser.py
 *                        cameras): per-frame intrinsics, OpenCV lens distortion, fisheye and equirectangular models
 *   fnr_tsdf_integrate, fnr_marching_cubes_scratch_bytes, fnr_marching_cubes_count, fnr_marching_cubes_emit
 *                        the `tsdf` mesh export (nerfstudio ns-export tsdf: TSDF.integrate_tsdf, skimage
 *                        marching_cubes): fusion of rendered depth maps and the scene / fruit surface meshes
 *   fnr_poisson_scratch_bytes, fnr_poisson_splat, fnr_poisson_apply, fnr_poisson_solve, fnr_poisson_sample
 *                        the `poisson` mesh export (nerfstudio ns-export poisson: open3d
 *                        create_from_point_cloud_poisson): screened Poisson reconstruction of the surface cloud
 *   fnr_mesh_measure_scratch_bytes, fnr_mesh_components, fnr_mesh_assign_centers, fnr_mesh_measure_groups
 *                        per-fruit measurement of the fruit meshes (no reference counterpart): grouping by connected
 *                        components or nearest count centre, area, sphere fit, volume, solid-angle coverage, edges
 *   fnr_image_metrics_scratch_bytes, fnr_image_stats, fnr_ssim
 *                        the `eval` command (nerfstudio ns-eval; FruitModel.get_image_metrics_and_images,
 *                        fruit_nerf/fruit_nerf.py:403-458): PSNR, SSIM and fruit-mask agreement of a rendered view
 *   fnr_texture_atlas_size, fnr_texel_rays, fnr_mesh_mean_edge
 *                        NeRF textures of the `tsdf` / `poisson` meshes (nerfstudio texture_utils.export_textured_mesh,
 *                        unwrap_method="custom"): the per-face UV atlas, one ray per texel, the ray length
 *   fnr_mesh_decimate_scratch_bytes, fnr_mesh_decimate
 *                        quadric edge-collapse decimation of the meshes before NeRF texturing (nerfstudio
 *                        target_num_faces; pymeshlab meshing_decimation_quadric_edge_collapse)
 *   fnr_chart_unwrap_scratch_bytes, fnr_chart_unwrap, fnr_chart_texel_rays
 *                        the `charts` UV unwrap of NeRF texturing (the project's own, in place of nerfstudio's xatlas):
 *                        area-proportional axis-projected charts packed into one square atlas, one ray per owned texel
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

/* fnr_pixel_batch for captured cameras (DESIGN.md section 4.3j): the same draws, gathers and outputs, with per-image
 * fx / fy / cx / cy [num_images] (DEVICE fp32, not NULL), optional distortion [num_images,6] = k1 k2 k3 k4 p1 p2 (DEVICE
 * fp32, or NULL for none) and camera_type FNR_CAMERA_* (defined below).  With (u, v) = ((x + 0.5 - cx) / fx,
 * -(y + 0.5 - cy) / fy) (fp32, correctly rounded divisions), (u, v) is undistorted by nerfstudio's
 * radial_and_tangential_undistort (10 Newton steps in fp64; not for equirectangular) and mapped to a direction as
 * fnr_camera_rays does.  Inputs are not checked for finiteness here: that is done once when the data set is loaded. */
int fnr_pixel_batch_lens(const float* rand, const float* c2w, const float* images, const float* masks, int32_t num_images,
                         int32_t height, int32_t width, const float* fx, const float* fy, const float* cx, const float* cy,
                         const float* distortion, int32_t camera_type, int32_t num_rays, float* origins, float* directions,
                         int32_t* camera_indices, int64_t* indices, float* image, float* fruit_mask, void* stream);

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

/* Bytes of caller-allocated device scratch fnr_render_backward needs for this shape and desc: the per-sample upstream
 * gradients (R*S*5 floats) for every impl, plus, for the fruit_nerf shape on the tensor-core impls, the level-major
 * encoding gradients (R*S*L*F floats, about 96 MiB at 4096 x 192) that its table scatter reads.  fnr_render_backward
 * refuses smaller scratch before any device work. */
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

/* counts[k*n + i] = fnr_radius_count(radius = radii[k], cap = caps[k]) counts[i], bit for bit, for k < num_radii, from
 * one grid whose cell side comes from the smallest radius (a larger radius walks the rings it needs): the outlier counts
 * of parameter sweeps (clustering.count_sweep).  radii / caps: HOST arrays of 1 <= num_radii <= 16 entries, every
 * radius positive and finite, every cap >= 1 (FNR_ERR_INVALID_ARGUMENT otherwise; more than 16 entries or a largest
 * radius more than 4 times the smallest return FNR_ERR_UNSUPPORTED).  The 2^21-cells-per-axis limit applies to the
 * smallest radius.  counts: DEVICE [num_radii, n] int32.  Scratch: fnr_cluster_scratch_bytes(n). */
int fnr_radius_count_multi(const double* points, int64_t num_points, const double* lo, const double* hi, const double* radii,
                           const int32_t* caps, int32_t num_radii, int32_t* counts, void* scratch, size_t scratch_bytes, void* stream);

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

/* ---- novel-view rendering (nerfstudio ns-render, the reference's debug/render.py launcher): camera rays of a camera
 * path made on the device chunk by chunk, and the per-frame uint8 image of the requested outputs (fnr_render.cu). ---- */

#define FNR_CAMERA_PERSPECTIVE 0
#define FNR_CAMERA_FISHEYE 1
#define FNR_CAMERA_EQUIRECTANGULAR 2

/* Rays of pixels [pixel_start, pixel_start + num_pixels) (row-major, pixel centres) of frame `frame` of a camera set:
 * c2w [num_frames,3,4] (OpenGL axes, DEVICE fp32), fx / fy / cx / cy [num_frames] (DEVICE fp64).  With
 * (u, v) = ((x + 0.5 - cx) / fx, -(y + 0.5 - cy) / fy) the camera-space direction is
 *   perspective      (u, v, -1)
 *   fisheye          (u sin(t) / t, v sin(t) / t, -cos(t)), t = min(|(u, v)|, pi); (0, 0, -1) at t = 0
 *   equirectangular  (-sin(a) sin(p), cos(p), -cos(a) sin(p)), a = -pi u, p = pi (0.5 - v)
 * then rotated and normalised in fp32 without FMA.  cx / cy are rounded to fp32, the divisions by fx / fy are multiplies
 * by fp32(1 / f) formed in fp64, and each 3-term sum is (a0 + a2) + a1: the op order torch's CUDA kernels give
 * synthetic_scene.camera_rays with python-float intrinsics, so perspective
 * rays are bit-identical to SyntheticCameras.generate_rays on the device.  origins / directions: DEVICE [num_pixels,3]
 * fp32. */
int fnr_camera_rays(const float* c2w, const double* fx, const double* fy, const double* cx, const double* cy, int32_t num_frames,
                    int32_t camera_type, int32_t height, int32_t width, int32_t frame, int64_t pixel_start, int32_t num_pixels,
                    float* origins, float* directions, void* stream);

/* fnr_camera_rays for the lens cameras of a data set: fx / fy / cx / cy [num_frames] (DEVICE fp32, not NULL), distortion
 * [num_frames,6] (DEVICE fp32, or NULL).  The arithmetic is fnr_pixel_batch_lens's (the pixel step a correctly rounded
 * division, 3-term sums left to right), so the ray of pixel (frame, y, x) is bit-identical to the training ray drawn for it. */
int fnr_camera_rays_lens(const float* c2w, const float* fx, const float* fy, const float* cx, const float* cy, const float* distortion,
                         int32_t num_frames, int32_t camera_type, int32_t height, int32_t width, int32_t frame, int64_t pixel_start,
                         int32_t num_pixels, float* origins, float* directions, void* stream);

#define FNR_MAX_FRAME_OUTPUTS 8
#define FNR_COMPOSE_PARTIALS 256
/* floats of the DEVICE scratch fnr_compose_frame needs when a depth output takes its near / far from the frame */
#define FNR_COMPOSE_SCRATCH_FLOATS (FNR_MAX_FRAME_OUTPUTS * FNR_COMPOSE_PARTIALS * 2)

#define FNR_FRAME_COLOR 0 /* [H*W,3] image shown as is (nerfstudio apply_colormap of a 3-channel image) */
#define FNR_FRAME_TURBO 1 /* [H*W] float through turbo: index long(clip(nan_to_num(v, 0), 0, 1) * 255) */
#define FNR_FRAME_DEPTH 2 /* [H*W] depth: apply_depth_colormap, clip((d - near) * fp32(1 / (far - near + 1e-10)), 0, 1)
                           * through turbo, then c * accumulation + (1 - accumulation) */
#define FNR_RANGE_AUTO_NEAR 1
#define FNR_RANGE_AUTO_FAR 2

typedef struct fnr_frame_output {
  const float* image;                /* DEVICE fp32, layout by kind */
  int32_t kind;                      /* FNR_FRAME_* */
  int32_t auto_range;                /* depth only, FNR_RANGE_AUTO_* bits: near / far taken from the frame's own min / max
                                      * (NaN if any depth is NaN, as torch.min / torch.max) */
  double near_plane, far_plane;      /* the others: near is rounded to fp32, far - near + 1e-10 is formed in fp64 */
} fnr_frame_output;

/* One frame of ns-render's _render_trajectory_video: the colour image of each output, side by side, quantised as
 * uint8(clip(x, 0, 1) * 255 + 0.5) (NaN -> 0) into image: DEVICE [height, width * num_outputs, 3] uint8.  accumulation:
 * DEVICE [H*W] fp32 (NULL: depth outputs are not blended).  turbo: DEVICE [256,3] fp32 colour table.  scratch: DEVICE
 * float[FNR_COMPOSE_SCRATCH_FLOATS] (NULL when no output uses auto_range).  Exact: min / max do not depend on order. */
int fnr_compose_frame(const fnr_frame_output* outputs, int32_t num_outputs, const float* accumulation, int32_t height, int32_t width,
                      const float* turbo, float* scratch, uint8_t* image, void* stream);

/* ---- Surface meshes (`ns-export-semantics tsdf`, nerfstudio ns-export tsdf; fnr_mesh.cu) ----
 * Grids are DEVICE fp32 in C order [nx, ny, nz] (z fastest); grid point (i,j,k) lies at origin + (i,j,k) * voxel_size per
 * axis (origin, voxel_size: HOST float[3]).  Every voxel, vertex and face count and index is int64.
 *
 * fnr_tsdf_integrate fuses num_frames rendered frames into the grid in place, frame after frame (no atomics: the result
 * does not depend on the launch).  State: values [N] (start at -1), weights [N] (start at 0; a plain count), colors
 * [N,3], fruit [N] (may be NULL when frame_fruit is).  Frames: c2w [B,3,4] (OpenGL axes), fx, fy, cx, cy [B], depth
 * [B,H,W] (the ray distance the model renders), rgb [B,H,W,3], frame_fruit [B,H,W] probabilities or NULL.  Per grid
 * point x and frame: p = R^T (x - t), z_c = -p.z (skip if <= 0); u = cx + fx p.x / z_c, v = cy - fy p.y / z_c; pixel
 * (floor u, floor v) (skip if off the image); the pixel's ray distance t becomes the depth
 * z = t / sqrt(((x + 0.5 - cx) / fx)^2 + ((y + 0.5 - cy) / fy)^2 + 1) of its centre ray; sdf = z - z_c (skip if t <= 0
 * or sdf <= -truncation); value, colour and fruit become (old * w + new) / (w + 1) with tsdf = clamp(sdf / truncation,
 * -1, 1), and w += 1.  FNR_ERR_INVALID_ARGUMENT: NULL state or inputs, a dim < 2, non-finite or non-positive voxel size
 * or truncation, H or W <= 0, num_frames < 0.  num_frames = 0 does nothing. */
int fnr_tsdf_integrate(float* values, float* weights, float* colors, float* fruit, int64_t nx, int64_t ny, int64_t nz, const float* origin,
                       const float* voxel_size, float truncation, const float* c2w, const float* fx, const float* fy, const float* cx,
                       const float* cy, const float* depth, const float* rgb, const float* frame_fruit, int32_t num_frames, int32_t height,
                       int32_t width, void* stream);

/* Marching cubes of values at level 0 (a corner is inside iff its value is < 0), in two passes around a host read of the
 * counts: fnr_marching_cubes_count fills DEVICE scratch (fnr_marching_cubes_scratch_bytes) and writes DEVICE
 * totals[2] = {vertices, faces}; fnr_marching_cubes_emit then writes vertices [V,3], unit normals [V,3] (the interpolated
 * central-difference gradient: toward increasing value; where it vanishes, the edge direction toward its outside end),
 * vertex_colors [V,3] / vertex_fruit [V] (the nearest grid
 * point's, round half to even; NULL exactly when colors / fruit is) and faces [F,3] int64.  Each grid edge with one
 * inside endpoint carries one vertex, ids in (point linear index, axis) order; faces run in cell order, then in the
 * order of the crack-free, orientable triangle table of fnr_mesh_table.h.  More than 2^31 - 1 vertices return
 * FNR_ERR_UNSUPPORTED (a PLY face list holds int indices). */
int fnr_marching_cubes_scratch_bytes(int64_t nx, int64_t ny, int64_t nz, size_t* bytes);
int fnr_marching_cubes_count(const float* values, int64_t nx, int64_t ny, int64_t nz, void* scratch, size_t scratch_bytes, int64_t* totals,
                             void* stream);
int fnr_marching_cubes_emit(const float* values, const float* colors, const float* fruit, int64_t nx, int64_t ny, int64_t nz, const float* origin,
                            const float* voxel_size, const void* scratch, size_t scratch_bytes, int64_t num_vertices, int64_t num_faces,
                            float* vertices, float* normals, float* vertex_colors, float* vertex_fruit, int64_t* faces, void* stream);

/* ---- Screened Poisson reconstruction (`ns-export-semantics poisson`, nerfstudio ns-export poisson; fnr_poisson.cu) ----
 * points: DEVICE [n,3] fp64, 1 <= n <= 2^31 - 1; normals [n,3], colors [n,3] (or NULL), fruit [n] (or NULL): DEVICE fp32.
 * The cube (origin: HOST double[3], side) carries R = 2^depth cells per axis, 2 <= depth <= 10, and (R+1)^3 nodes in C
 * order; node (i,j,k) lies at origin + (i,j,k) * side / R.  Every point must be finite and lie in a cell,
 * 0 <= floor((p - origin) / (side / R)) < R per axis (FNR_ERR_INVALID_ARGUMENT otherwise: one host read).  Node sums
 * gather over the points of the node's 8 adjacent cells, in cell order and then input order, in fp64 rounded to fp32
 * once (no atomics: repeated calls give identical bits).  DEVICE scratch: fnr_poisson_scratch_bytes(n, depth).
 *
 * fnr_poisson_splat writes density [M] = sum phi, normal_field [M,3] = (a / h^3) sum phi n with h = 1/R and
 * a = h^2 * (occupied cells) / n, node_colors [M,3] / node_fruit [M] = sum phi c / density (0 where density is 0; NULL
 * exactly when colors / fruit is) and rhs [M] = sum_j (int grad phi_i phi_j) . v_j.  It leaves the sorted points in
 * scratch, which fnr_poisson_apply reads: y = (K + alpha a S^T S) x for x [M], with K the Q1 stiffness matrix of the
 * cells inside the cube (Neumann boundaries) and S [n, M] the trilinear point samples.
 * fnr_poisson_solve splats at every depth from max(depth - 3, 4) to depth (depth alone when depth <= 4) and solves each
 * level by Jacobi-preconditioned conjugate gradient in fp32 (fp64 block dot products), starting from the previous
 * level's chi prolonged trilinearly, until |r| <= tolerance |b| or max_iters iterations.  chi [M]; density,
 * node_colors, node_fruit as fnr_poisson_splat's at the finest depth; HOST iterations[2] = {finest level, all levels};
 * HOST residual = |r| / |b| at the finest level.
 * fnr_poisson_sample writes out [n] fp32, the trilinear sample of a node grid [M] at each point (clamped to the border
 * cells). */
int fnr_poisson_scratch_bytes(int64_t num_points, int32_t depth, size_t* bytes);
int fnr_poisson_splat(const double* points, const float* normals, const float* colors, const float* fruit, int64_t num_points, int32_t depth,
                      const double* origin, double side, void* scratch, size_t scratch_bytes, float* density, float* normal_field,
                      float* node_colors, float* node_fruit, float* rhs, void* stream);
int fnr_poisson_apply(int64_t num_points, int32_t depth, float alpha, const void* scratch, size_t scratch_bytes, const float* x, float* y,
                      void* stream);
int fnr_poisson_solve(const double* points, const float* normals, const float* colors, const float* fruit, int64_t num_points, int32_t depth,
                      const double* origin, double side, float alpha, int32_t max_iters, float tolerance, void* scratch, size_t scratch_bytes,
                      float* chi, float* density, float* node_colors, float* node_fruit, int64_t* iterations, double* residual, void* stream);
int fnr_poisson_sample(const double* points, int64_t num_points, int32_t depth, const double* origin, double side, const float* grid, float* out,
                       void* stream);

/* ---- Per-fruit measurement of triangle meshes (fnr_measure.cu; DESIGN section 4.3n) ----
 * vertices: DEVICE [V,3] fp64; faces: DEVICE [F,3] int64, every index in [0, V) (FNR_ERR_INVALID_ARGUMENT otherwise: a
 * device check and one host read); face_group: DEVICE [F] int32, a group id or -1 (unassigned).  V <= 2^31 - 1 and
 * F <= (2^31 - 1) / 3, else FNR_ERR_UNSUPPORTED; negative counts and NULL inputs return FNR_ERR_INVALID_ARGUMENT.
 * DEVICE scratch of fnr_mesh_components and fnr_mesh_measure_groups: fnr_mesh_measure_scratch_bytes(V, F).
 *
 * fnr_mesh_components labels each face with its connected component (faces connected when they share a vertex index;
 * vertices no face uses are ignored), components numbered in the order of their smallest vertex index, and writes the
 * count to HOST *num_groups (one host read).
 * fnr_mesh_assign_centers labels each face with the index of the centre (DEVICE [K,3] fp64, all finite) nearest its
 * centroid (v0 + v1 + v2) / 3 in fp64 squared distance ((dx^2 + dy^2) + dz^2, no FMA; ties to the lower index), or -1
 * when that distance exceeds max_distance (> 0; may be infinite).  Its DEVICE scratch is FNR_MESH_ASSIGN_SCRATCH_BYTES
 * (the flag of the check of the face indices and the centres, one host read).
 * fnr_mesh_measure_groups measures the groups 0..G-1 (labels outside [-1, G) are refused).  Per group: group_faces,
 * boundary_edges, nonmanifold_edges [G] int64 (per edge key (min, max) vertex id and group: one half-edge of the group is
 * a boundary edge, three or more a non-manifold edge); area [G] = sum |e1 x e2| / 2; centroid [G,3] area-weighted (the
 * plain mean of the face centroids when the area is 0); sphere [G,5] = centre xyz, radius and area-weighted RMS of
 * |p_f - centre| - radius over the face centroids p_f, from the area-weighted algebraic (Kasa) fit about the centroid;
 * fit_ok [G] int32 (0: singular system or d + |x|^2 <= 0, centre = centroid, radius = the area-weighted RMS distance of
 * the face centroids from it); volume [G] = sum det(v0 - c, v1 - c, v2 - c) / 6 and coverage [G] = (sum of the signed
 * solid angles, Van Oosterom-Strackee) / 4 pi, about c = the sphere centre; both are positive for faces whose right-hand
 * normal points out of the enclosed volume.  A group with no faces gets 0 counts, area, volume and coverage and NaN
 * centroid and sphere.  unassigned_faces [1] / unassigned_area [1] (DEVICE, both or neither NULL): the label -1 faces.
 * Every sum runs in a fixed order: repeated calls give identical bits. */
int fnr_mesh_measure_scratch_bytes(int64_t num_vertices, int64_t num_faces, size_t* bytes);
int fnr_mesh_components(const int64_t* faces, int64_t num_faces, int64_t num_vertices, void* scratch, size_t scratch_bytes, int32_t* face_group,
                        int64_t* num_groups, void* stream);
#define FNR_MESH_ASSIGN_SCRATCH_BYTES 256
int fnr_mesh_assign_centers(const double* vertices, const int64_t* faces, int64_t num_faces, int64_t num_vertices, const double* centers,
                            int64_t num_centers, double max_distance, void* scratch, size_t scratch_bytes, int32_t* face_group, void* stream);
int fnr_mesh_measure_groups(const double* vertices, const int64_t* faces, int64_t num_faces, int64_t num_vertices, const int32_t* face_group,
                            int64_t num_groups, void* scratch, size_t scratch_bytes, int64_t* group_faces, int64_t* boundary_edges,
                            int64_t* nonmanifold_edges, double* area, double* centroid, double* sphere, double* volume, double* coverage,
                            int32_t* fit_ok, int64_t* unassigned_faces, double* unassigned_area, void* stream);

/* ---- Held-out evaluation scores of one rendered view (the `eval` command, nerfstudio ns-eval; fnr_metrics.cu; DESIGN
 * section 4.3o) ----
 * rgb: DEVICE [H*W,3] fp32 as rendered (clamped to [0,1] here, as FruitModel.get_image_metrics_and_images does; NaN stays
 * NaN); semantics [H*W] logits, accumulation [H*W], image [H,W,3] and fruit_mask [H*W] ({0,1}): DEVICE fp32.
 * 1 <= H*W <= (2^31 - 1) / 3.  record: DEVICE double[FNR_IMAGE_RECORD_DOUBLES], slots FNR_REC_*; the counts are whole
 * numbers held exactly in fp64.  DEVICE scratch: fnr_image_metrics_scratch_bytes(H, W), shared by the two calls of one
 * image.  Sums are fp64 block sums in a fixed tree, finished in index order over a grid that depends on H and W alone:
 * no floating-point atomics, and repeated calls give identical bits.
 *
 * fnr_image_stats writes slots SSE .. FRUIT_TN: the sum over the 3 H W values of (clamp(rgb) - image)^2 (PSNR is
 * 10 log10(3 H W / SSE)); min / max of clamp(rgb) and of image (NaN ignored); the sum of accumulation; the confusion
 * counts of fp32 sigmoid(semantics) > 0.9 (the thresholding of FruitModel.get_outputs) against fruit_mask > 0.5.
 * fnr_ssim reads the four min / max slots, so it follows fnr_image_stats of the same image on the stream, and writes
 * slots SSIM and DATA_RANGE: torchmetrics structural_similarity_index_measure with its defaults (11x11 gaussian window,
 * sigma 1.5, k1 0.01, k2 0.03, data_range = the larger fp32 value range of the two images, the map cropped by 5 pixels
 * per side and averaged over pixels and channels), window sums and formula in fp64.  The crop keeps only windows that
 * lie inside the image, so torchmetrics' reflect padding never reaches a kept pixel and none is applied.  H or W < 11
 * (an empty cropped map) returns FNR_ERR_UNSUPPORTED. */
#define FNR_IMAGE_RECORD_DOUBLES 12
#define FNR_IMAGE_STATS_PARTIALS 256
#define FNR_REC_SSE 0
#define FNR_REC_RGB_MIN 1
#define FNR_REC_RGB_MAX 2
#define FNR_REC_IMAGE_MIN 3
#define FNR_REC_IMAGE_MAX 4
#define FNR_REC_ACCUMULATION_SUM 5
#define FNR_REC_FRUIT_TP 6
#define FNR_REC_FRUIT_FP 7
#define FNR_REC_FRUIT_FN 8
#define FNR_REC_FRUIT_TN 9
#define FNR_REC_SSIM 10
#define FNR_REC_DATA_RANGE 11
int fnr_image_metrics_scratch_bytes(int32_t height, int32_t width, size_t* bytes);
int fnr_image_stats(const float* rgb, const float* semantics, const float* accumulation, const float* image, const float* fruit_mask,
                    int32_t height, int32_t width, void* scratch, size_t scratch_bytes, double* record, void* stream);
int fnr_ssim(const float* rgb, const float* image, int32_t height, int32_t width, void* scratch, size_t scratch_bytes, double* record,
             void* stream);

/* ---- NeRF textures of exported meshes (`--texture-method nerf --unwrap-method custom`, nerfstudio
 * texture_utils.export_textured_mesh with unwrap_method="custom"; fnr_texture.cu; DESIGN section 4.3p) ----
 * The atlas of F faces at p = px_per_uv_triangle texels per triangle (2 <= p, 1 <= F <= FNR_TEXTURE_MAX_FACES): blocks
 * of p rows by p + 3 columns, two faces each (faces 2k and 2k + 1 in block k), blocks row-major, bx per row, where bx is
 * the smallest b >= 1 with b^2 (p + 3) >= ceil(F / 2) p.  width = bx (p + 3), height = ceil(ceil(F / 2) / bx) p; a side over
 * FNR_TEXTURE_MAX_SIDE is refused.  Texel (row, col), row 0 at the top (OBJ v = 1 - (row + 0.5) / height), lies in block
 * (row / p) bx + col / (p + 3) at (a, b) = (col % (p + 3), row % p); it belongs to slot 2 block + (a + b >= p + 1), whose
 * frame coordinates are (a, b) for the first slot and (p + 2 - a, p - 1 - b) for the second.  In its frame a slot's UV
 * triangle has its face's vertices 0, 1, 2 at the texel centres (0, 0), (p - 1, 0), (0, p - 1).  A bilinear lookup inside
 * the triangle reads only texels of its own slot, and slots >= F (after the last face) are never sampled; their texels
 * take the rays of face F - 1.
 *
 * fnr_texel_rays writes the rays of texels [texel_start, texel_start + num_texels) (row-major) of that atlas: vertices,
 * normals DEVICE [V,3] fp32; faces DEVICE [F,3] int64, every index in [0, V) (not checked); origins, directions DEVICE
 * [num_texels,3] fp32.  Per texel, in fp32 without FMA: the frame coordinates (la, lb) give the closest point (xs, ys) of
 * the triangle, (la, lb) itself when la + lb <= p - 1, else xs = clamp(la - 0.5, 0, p - 1), ys = (p - 1) - xs;
 * s = xs / (p - 1), t = ys / (p - 1), w0 = (1 - s) - t; x = (w0 v0 + s v1) + t v2 and n = (w0 n0 + s n1) + t n2 per
 * component; |n| = sqrt((n.x^2 + n.y^2) + n.z^2).  When |n| > 1e-12 fails, n is the face normal (v1 - v0) x (v2 - v0)
 * (each component a rounded difference of rounded products), and when that fails too, (0, 0, 1).  With n_k = n_k / |n|:
 * direction = -n, origin_k = x_k + (0.5 raylen) n_k.  The rays are nerfstudio's: origin 0.5 raylen outside the surface,
 * nears 0 and fars raylen (set by the caller).  FNR_ERR_INVALID_ARGUMENT: a NULL pointer, p < 2, F < 1, a width / height
 * other than the layout's, a texel range outside [0, width * height), a raylen that is not finite and positive.
 *
 * fnr_mesh_mean_edge writes out[0] = the mean over faces of |v1 - v0| (fp64 differences of the fp32 vertices, sum
 * (d.x^2 + d.y^2) + d.z^2, no FMA): block b of FNR_MEAN_EDGE_PARTIALS sums faces [b per, (b + 1) per), per =
 * ceil(F / FNR_MEAN_EDGE_PARTIALS), into out[1 + b] in a fixed tree, and one finish adds the partials in a fixed tree.  No
 * atomics: repeated calls give identical bits.  out: DEVICE double[FNR_MEAN_EDGE_DOUBLES].
 *
 * fnr_texture_atlas_size writes the layout's HOST width and height (also when a side exceeds FNR_TEXTURE_MAX_SIDE). */
#define FNR_TEXTURE_MAX_SIDE 16384
#define FNR_TEXTURE_MAX_FACES (2LL * FNR_TEXTURE_MAX_SIDE * FNR_TEXTURE_MAX_SIDE)
#define FNR_MEAN_EDGE_PARTIALS 256
#define FNR_MEAN_EDGE_DOUBLES (1 + FNR_MEAN_EDGE_PARTIALS)
int fnr_texture_atlas_size(int64_t num_faces, int32_t px_per_uv_triangle, int64_t* width, int64_t* height);
int fnr_texel_rays(const float* vertices, const float* normals, const int64_t* faces, int64_t num_faces, int32_t px_per_uv_triangle,
                   int32_t width, int32_t height, float raylen, int64_t texel_start, int32_t num_texels, float* origins, float* directions,
                   void* stream);
int fnr_mesh_mean_edge(const float* vertices, const int64_t* faces, int64_t num_faces, double* out, void* stream);

/* ---- Quadric edge-collapse decimation (`--target-num-faces` of the tsdf / poisson exports with NeRF texturing;
 * fnr_decimate.cu; DESIGN section 4.3q) ----
 * vertices: DEVICE [V,3] fp64; faces: DEVICE [F,3] int64, every index in [0, V) (FNR_ERR_INVALID_ARGUMENT otherwise: a
 * device check and one host read).  V <= 2^31 - 1 and F <= (2^31 - 1) / 3, else FNR_ERR_UNSUPPORTED; NULL pointers,
 * negative counts and target_num_faces < 1 return FNR_ERR_INVALID_ARGUMENT.  DEVICE scratch:
 * fnr_mesh_decimate_scratch_bytes(V, F); nothing is allocated.  Outputs sized to the input: out_vertices,
 * out_normals DEVICE [V,3] fp64, out_faces DEVICE [F,3] int64, of which the first HOST *out_num_vertices /
 * *out_num_faces rows are written; HOST *out_rounds counts the rounds that collapsed edges.
 *
 * In this order, every fp64 operation rounded where written (no FMA; decimate.py restates it bit for bit):
 *  1. Quadrics (10 entries xx xy xz xw yy yz yw zz zw ww, each w * (p_i * p_j) of a plane p = (u, -u.x)).  Face f with
 *     n = (v1 - v0) x (v2 - v0): the plane u = n / |n| through v0, w = |n| / 2.  Each boundary half-edge (its edge in
 *     one face) from corner k to k + 1, e = v_k+1 - v_k: the plane u = (e x n) / |e x n| through v_k, w = 100 |e|^2.
 *     A plane with a zero normal adds nothing.  Corner (f, k) adds the face plane, then the boundary planes of
 *     half-edges k and k + 2; a vertex sums its corners in face order, from 0.
 *  2. Each round, on the faces as they stand: the 3F half-edge keys min * V + max and the corners by vertex, each
 *     stably radix-sorted.  An edge (a < b) is a run of equal keys; it is valid when it is in 1 or 2 faces, a != b,
 *     |N(a) & N(b)| equals its face count, it is not in 2 faces with both ends on a boundary edge, in 2 faces its
 *     opposite vertices differ and share no face, and every face around a or b not holding both keeps
 *     dot(n_old, n_new) > 0 with a and b moved to the placement.
 *  3. Placement: Gaussian elimination with partial pivoting (first largest |pivot|) of the 3x3 system of Q = Q_a + Q_b;
 *     when a pivot is not above 1e-8 times the largest |diagonal|, the best of v_a, v_b and (v_a + v_b) * 0.5 (ties
 *     in that order).  Cost = v^T Q v as ((x r0 + y r1) + z r2) + r3, r_i = ((q_i0 x + q_i1 y) + q_i2 z) + q_i3,
 *     clamped at 0.
 *  4. Rank = position in a stable sort of the valid edges by the cost's bits (edge order breaks ties); m1[v] = the
 *     least rank at v, m2[v] = the least m1 over v and its neighbours; an edge is selected when rank = m2[a] = m2[b]
 *     (selected edges share no face).  In rank order, a selected edge collapses while the face count before it is
 *     above target + 1: v_a = the placement, Q_a = Q_a + Q_b, b -> a; faces with a repeated index are dropped, the
 *     rest kept in order.
 *  5. Rounds end when F <= target + 1 or when a round finds no valid edge (F is then returned as it stands).
 *  6. Vertices no face uses are dropped in input order; normals = s / |s| with s the sum, in face order, of the
 *     vertex's (v1 - v0) x (v2 - v0); 0 where s = 0.  One host read per round. */
int fnr_mesh_decimate_scratch_bytes(int64_t num_vertices, int64_t num_faces, size_t* bytes);
int fnr_mesh_decimate(const double* vertices, const int64_t* faces, int64_t num_vertices, int64_t num_faces, int64_t target_num_faces,
                      void* scratch, size_t scratch_bytes, double* out_vertices, double* out_normals, int64_t* out_faces,
                      int64_t* out_num_vertices, int64_t* out_num_faces, int32_t* out_rounds, void* stream);

/* ---- The `charts` UV unwrap (`--unwrap-method charts` of NeRF texturing; fnr_unwrap.cu, fnr_texture.cu; DESIGN section
 * 4.3r) ----
 * vertices: DEVICE [V,3] fp32, finite; faces: DEVICE [F,3] int64, every index in [0, V) (FNR_ERR_INVALID_ARGUMENT
 * otherwise: a device check and one host read).  N = num_pixels_per_side in [FNR_UNWRAP_MIN_SIDE, FNR_TEXTURE_MAX_SIDE],
 * V >= 1, F >= 1 and no NULL pointer (stage_ms aside), else FNR_ERR_INVALID_ARGUMENT before any CUDA call; V > 2^31 - 1
 * or F > (2^31 - 1) / 3: FNR_ERR_UNSUPPORTED.  DEVICE scratch: fnr_chart_unwrap_scratch_bytes(V, F, N); nothing is
 * allocated on the device.  Outputs, DEVICE: labels, charts [F] int32; offsets [F,2] int32 (the first C rows written);
 * uv [F,3,2] fp64; owner [N*N] int32; texels, texel_faces [N*N] int32 and barycentrics [N*N,3] fp32 (the first
 * *out_num_owned rows written).  HOST: *out_rounds, *out_num_charts (C), *out_scale (s), *out_num_owned; stage_ms, when
 * not NULL, HOST double[FNR_UNWRAP_STAGES] of wall milliseconds (labels and edge sort, charts, packing, raster and
 * conflicts, owners and compaction; the stream is drained at each stage boundary).
 *
 * In this order, every fp64 operation rounded where written (no FMA; texture.py restates it bit for bit):
 *  1. Positions P = (double)v + 0.  Face f: e1 = P1 - P0, e2 = P2 - P0, n = e1 x e2 (each component a rounded difference
 *     of rounded products).  Its label is 2k + (n_k < 0) for the axis k of the largest |n_k|, ties to the lower axis (a
 *     zero normal gets +x, label 0).  Projected corner p = (P[a], P[b]) with (a, b) = (z, y), (y, z), (x, z), (z, x),
 *     (y, x), (x, y) for the labels +x, -x, +y, -y, +z, -z: a face has negative area in texel space (x right, y down) and
 *     positive area in vt space.
 *  2. Charts.  The 3F half-edges (fnr_mesh_edges.cuh) sorted once; a run of exactly two half-edges joins their faces when
 *     the labels are equal and neither face is cut.  Chart id = rank of the chart's smallest face index.
 *  3. Extents per chart and axis: ext = max - min of its projected corners, p_min = min.
 *  4. Packing, on the host: charts sorted by (ext_y desc, ext_x desc, id asc); at scale s a chart's rectangle is
 *     floor(s ext_x) + 1 + 2 FNR_UNWRAP_MARGIN by floor(s ext_y) + 1 + 2 FNR_UNWRAP_MARGIN texels, placed by next-fit shelves
 *     (a rectangle that overflows the row opens a shelf below the tallest of the row) into N x N; offsets = its top-left
 *     texel.  When s = 0 does not pack, *out_scale = -1 and nothing after this step is written.  Otherwise, with E the
 *     largest extent, s = 0 when E = 0, else lo = 0, hi = N / E and FNR_UNWRAP_BISECTIONS steps mid = (lo + hi) * 0.5,
 *     lo = mid when it packs, else hi = mid; s = lo.
 *  5. Texel coordinates of corner (f, k): x = (double)(offset_x + FNR_UNWRAP_MARGIN) + s * (p_x - p_min,x), likewise y.
 *     vt = (x / N, 1 - y / N).  Texel (row, col) has its centre at (col + 0.5, row + 0.5).
 *  6. Edge function of edge a -> b at c: (c_x - a_x) * (b_y - a_y) - (c_y - a_y) * (b_x - a_x); e_0, e_1, e_2 of the edges
 *     1 -> 2, 2 -> 0, 0 -> 1.  A texel centre is strictly inside when all three are > 0.  A texel centre strictly inside two
 *     triangles is a conflict: every face there but the smallest becomes cut (a chart of its own), and steps 2 to 6 run
 *     again; *out_rounds counts the rounds that cut a face.
 *  7. Owners.  Per face, every texel whose centre lies within FNR_UNWRAP_GUTTER of its texel box [min - g, max + g] per
 *     axis, clamped to the atlas: the squared distance d2 to the triangle is 0 when e_0, e_1, e_2 >= 0 and
 *     sum = (e_0 + e_1) + e_2 > 0, else the least over the edges k -> k + 1 (k = 0, 1, 2, ties to the lower k) of
 *     |c - (a + t (b - a))|^2 (x^2 + y^2), t = clamp(((c_x - a_x) d_x + (c_y - a_y) d_y) / |d|^2, 0, 1) with d = b - a,
 *     t = 0 when |d|^2 = 0.  When d2 <= g^2, atomicMin of (fp32(d2) bits << 32) | f: the winner owns the texel.
 *     Barycentrics (fp32) of the owner's closest point: inside, w1 = fp32(e_1 / sum), w2 = fp32(e_2 / sum),
 *     w0 = max((1 - w1) - w2, 0); on edge k, w_k = 1 - fp32(t), w_k+1 = fp32(t), the third 0; when sum <= 0 (a degenerate
 *     triangle), (1, 0, 0).  owner = the face or -1; the owned texels are compacted in texel order.
 *
 * fnr_chart_texel_rays writes the rays of owned texels [texel_start, texel_start + num_texels) of num_owned (texel_faces,
 * barycentrics as fnr_chart_unwrap wrote them) into origins, directions DEVICE [num_texels,3] fp32, with fnr_texel_rays'
 * arithmetic after its barycentrics.  FNR_ERR_INVALID_ARGUMENT: a NULL pointer, F < 1, a range outside [0, num_owned), a
 * raylen that is not finite and positive. */
#define FNR_UNWRAP_MIN_SIDE 16
#define FNR_UNWRAP_MARGIN 3
#define FNR_UNWRAP_GUTTER 2
#define FNR_UNWRAP_BISECTIONS 40
#define FNR_UNWRAP_STAGES 5
int fnr_chart_unwrap_scratch_bytes(int64_t num_vertices, int64_t num_faces, int32_t num_pixels_per_side, size_t* bytes);
int fnr_chart_unwrap(const float* vertices, const int64_t* faces, int64_t num_vertices, int64_t num_faces, int32_t num_pixels_per_side,
                     void* scratch, size_t scratch_bytes, int32_t* labels, int32_t* charts, int32_t* offsets, double* uv, int32_t* owner,
                     int32_t* texels, int32_t* texel_faces, float* barycentrics, int32_t* out_rounds, int64_t* out_num_charts,
                     double* out_scale, int64_t* out_num_owned, double* stage_ms, void* stream);
int fnr_chart_texel_rays(const float* vertices, const float* normals, const int64_t* faces, int64_t num_faces, const int32_t* texel_faces,
                         const float* barycentrics, int64_t num_owned, float raylen, int64_t texel_start, int32_t num_texels, float* origins,
                         float* directions, void* stream);

/* Hash-grid row indices (exact-integer parity hook): rows[N,L,8] in nerfstudio corner order for
 * the masked [0,1]^3 positions of the given samples; also writes positions[N,3] if non-NULL. */
int fnr_hash_indices(const fnr_field_desc* desc, const fnr_ray_batch* rays, int32_t* rows, float* positions,
                     void* stream);

/* The tensor-core backward's table-gradient scatter on its own (test hook): for every level l and sample p, adds
 * denc[l][p] (float2, level-major [L][N], N = num_rays * num_samples) times each corner's trilinear weight to the
 * corner's row of table_grad [L * 2^log2T, 2] (16-byte aligned), at the masked positions of the given samples.
 * features_per_level must be 2. */
int fnr_level_scatter(const fnr_field_desc* desc, const fnr_ray_batch* rays, const float* denc, float* table_grad,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FRUITNERF_B200_H */
