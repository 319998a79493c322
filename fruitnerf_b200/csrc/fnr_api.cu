// extern "C" entry points of libfruitnerf_b200.so: argument validation, conversion of the plain-C
// structs of include/fruitnerf_b200.h into kernel arguments, dispatch between the tensor-core
// (wgmma) and the fp32 simt instantiations of the field kernels.  No host synchronisation, no allocation.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return FNR_OK;
  set_error("CUDA error in %s: %s", what, cudaGetErrorString(e));
  return FNR_ERR_CUDA;
}

// every kernel launch of the library ends here: launch counter (fnr_launch_count) + launch-error check
static std::atomic<unsigned long long> g_launches{0};
int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_cuda(cudaGetLastError(), what);
}

static bool mlp_is(const fnr_mlp_desc& m, int n, const int* dims) {
  if (m.n_layers != n) return false;
  for (int i = 0; i <= n; ++i)
    if (m.dims[i] != dims[i]) return false;
  return true;
}

Family classify(const fnr_field_desc* d) {
  if (d->num_levels != 16 || d->features_per_level != 2 || d->appearance_dim != 32) return kFamilyNone;
  {
    const int base[] = {32, 64, 16}, sem[] = {15, 64, 64}, col[] = {63, 64, 64, 3};
    if (d->geo_feat_dim == 15 && mlp_is(d->base, 2, base) && mlp_is(d->semantic, 2, sem) && mlp_is(d->color, 3, col))
      return kFamilySmall;
  }
  {
    const int base[] = {32, 64, 31}, sem[] = {30, 128, 128, 64}, col[] = {78, 64, 64, 3};
    if (d->geo_feat_dim == 30 && mlp_is(d->base, 2, base) && mlp_is(d->semantic, 3, sem) && mlp_is(d->color, 3, col))
      return kFamilyBig;
  }
  return kFamilyNone;
}

int validate_desc(const fnr_field_desc* d) {
  if (!d) {
    set_error("desc is NULL");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (d->num_levels < 1 || d->num_levels > FNR_MAX_LEVELS || d->log2_hashmap_size < 1 || d->log2_hashmap_size > 26) {
    set_error("invalid hash grid (L=%d, T=%d)", d->num_levels, d->log2_hashmap_size);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if ((long long)d->num_levels << d->log2_hashmap_size > 0x7fffffffLL) {
    set_error("hash table rows exceed int32");
    return FNR_ERR_UNSUPPORTED;
  }
  if (d->position_mode != FNR_POS_CONTRACT && d->position_mode != FNR_POS_AABB) {
    set_error("invalid position_mode %d", d->position_mode);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (d->appearance_mode < FNR_APP_PER_CAMERA || d->appearance_mode > FNR_APP_ZEROS) {
    set_error("invalid appearance_mode %d", d->appearance_mode);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (d->num_images < 1) {
    set_error("num_images must be >= 1");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  // AUTO runs the tensor-core kernels like TCGEN05 (tc = impl != SIMT): every shape that passes validation is a shipped family
  if (d->impl != FNR_IMPL_AUTO && d->impl != FNR_IMPL_SIMT && d->impl != FNR_IMPL_TCGEN05) {
    set_error("invalid impl %d", d->impl);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (classify(d) == kFamilyNone) {
    set_error(
        "unsupported FruitField shape: kernels are specialised for fruit_nerf (geo 15, semantic 15-64-64, colour "
        "63-64-64-3) and fruit_nerf_big/_huge (geo 30, semantic 30-128-128-64, colour 78-64-64-3) with L=16, F=2, "
        "appearance 32");
    return FNR_ERR_UNSUPPORTED;
  }
  return FNR_OK;
}

static KField make_field(const fnr_field_desc* d) {
  KField F;
  F.L = d->num_levels;
  F.log2T = d->log2_hashmap_size;
  F.num_images = d->num_images;
  F.position_mode = d->position_mode;
  F.appearance_mode = d->appearance_mode;
  F.pass_semantic_gradients = d->pass_semantic_gradients;
  memcpy(F.scalings, d->scalings, sizeof(F.scalings));
  memcpy(F.aabb, d->aabb, sizeof(F.aabb));
  return F;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static int make_params(const fnr_field_desc* d, const fnr_field_params* p, KParams* K, const char* what) {
  if (!p) {
    set_error("%s is NULL", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  memset(K, 0, sizeof(*K));
  K->hash_table = p->hash_table;
  K->head_w = p->head_w;
  K->head_b = p->head_b;
  K->app_embedding = p->app_embedding;
  bool ok = p->hash_table && p->head_w && p->head_b && p->app_embedding && aligned16(p->hash_table) && aligned16(p->head_w);
  for (int i = 0; i < d->base.n_layers; ++i) {
    K->base_w[i] = p->base_w[i];
    K->base_b[i] = p->base_b[i];
    ok = ok && p->base_w[i] && p->base_b[i] && aligned16(p->base_w[i]);
  }
  for (int i = 0; i < d->semantic.n_layers; ++i) {
    K->sem_w[i] = p->sem_w[i];
    K->sem_b[i] = p->sem_b[i];
    ok = ok && p->sem_w[i] && p->sem_b[i] && aligned16(p->sem_w[i]);
  }
  for (int i = 0; i < d->color.n_layers; ++i) {
    K->col_w[i] = p->col_w[i];
    K->col_b[i] = p->col_b[i];
    ok = ok && p->col_w[i] && p->col_b[i] && aligned16(p->col_w[i]);
  }
  if (!ok) {
    set_error("%s: NULL or non-16-byte-aligned parameter pointer", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  return FNR_OK;
}

static int make_rays(const fnr_field_desc* d, const fnr_ray_batch* r, KRays* K) {
  if (!r) {
    set_error("rays is NULL");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (r->num_rays < 0 || r->num_samples < 1) {
    set_error("invalid ray batch shape R=%d S=%d", r->num_rays, r->num_samples);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (r->num_rays > 0 && (!r->origins || !r->directions || !r->starts || !r->ends)) {
    set_error("ray batch has NULL origins/directions/starts/ends");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (r->num_rays > 0 && d->appearance_mode == FNR_APP_PER_CAMERA && !r->camera_indices) {
    set_error("Camera indices are not provided.");  // fruit_field.py:240-241
    return FNR_ERR_INVALID_ARGUMENT;
  }
  K->R = r->num_rays;
  K->S = r->num_samples;
  K->origins = r->origins;
  K->directions = r->directions;
  K->starts = r->starts;
  K->ends = r->ends;
  K->camera_indices = r->camera_indices;
  return FNR_OK;
}

}  // namespace fnr

using namespace fnr;

extern "C" {

int fnr_version(void) { return FNR_ABI_VERSION; }

uint64_t fnr_launch_count(int32_t reset) {
  return reset ? fnr::g_launches.exchange(0, std::memory_order_relaxed) : fnr::g_launches.load(std::memory_order_relaxed);
}

const char* fnr_last_error(void) { return g_error; }

int fnr_render_forward(const fnr_field_desc* desc, const fnr_field_params* params, const fnr_ray_batch* rays,
                       const fnr_render_out* out, void* stream) {
  int rc = validate_desc(desc);
  if (rc) return rc;
  KParams P;
  KRays Rr;
  if ((rc = make_params(desc, params, &P, "params"))) return rc;
  if ((rc = make_rays(desc, rays, &Rr))) return rc;
  if (!out) {
    set_error("out is NULL");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (out->stash_encoding && (reinterpret_cast<uintptr_t>(out->stash_encoding) & 31u)) {
    set_error("stash_encoding must be 32-byte aligned (written with 256-bit stores)");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const bool composite = out->rgb || out->accumulation || out->depth || out->depth_index || out->semantics || out->weights;
  if (composite && !(out->sample_density && out->sample_rgb && out->sample_semantics)) {
    set_error("render: sample_density/sample_rgb/sample_semantics buffers are required when ray outputs are requested");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const bool tc = desc->impl != FNR_IMPL_SIMT;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  KFieldOut O{out->sample_density, out->sample_rgb, out->sample_semantics, out->stash_encoding};
  if ((rc = launch_field_forward(classify(desc), tc, make_field(desc), P, Rr, O, st))) return rc;
  if (!composite) return FNR_OK;
  KComposite Cm{out->sample_density, out->sample_rgb, out->sample_semantics, out->rgb, out->accumulation, out->depth,
                out->depth_index, out->semantics, out->weights, out->clamp_rgb};
  return launch_simt_composite(Rr, Cm, st);
}

int fnr_render_backward_scratch_bytes(const fnr_field_desc* desc, int32_t num_rays, int32_t num_samples, size_t* bytes) {
  int rc = validate_desc(desc);
  if (rc) return rc;
  if (!bytes || num_rays < 0 || num_samples < 1) {
    set_error("invalid arguments to fnr_render_backward_scratch_bytes");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  *bytes = (size_t)num_rays * num_samples * 5 * sizeof(float) + 256;
  return FNR_OK;
}

int fnr_render_backward(const fnr_field_desc* desc, const fnr_field_params* params, const fnr_ray_batch* rays,
                        const fnr_render_saved* saved, const fnr_render_grads* up, const fnr_field_params* grads,
                        void* scratch, size_t scratch_bytes, void* stream) {
  int rc = validate_desc(desc);
  if (rc) return rc;
  KParams P, G;
  KRays Rr;
  if ((rc = make_params(desc, params, &P, "params"))) return rc;
  if ((rc = make_params(desc, grads, &G, "grads"))) return rc;
  if ((rc = make_rays(desc, rays, &Rr))) return rc;
  if (!saved || !up) {
    set_error("saved/upstream is NULL");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (Rr.R == 0) return FNR_OK;
  // saved->weights == NULL selects the field-only backward (upstream = d_sample_* only)
  if (saved->weights && (!saved->sample_density || !saved->sample_rgb || !saved->sample_semantics || !saved->accumulation)) {
    set_error("saved forward products (sample_*, accumulation) are required next to weights");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  size_t need = 0;
  fnr_render_backward_scratch_bytes(desc, Rr.R, Rr.S, &need);
  if (!scratch || scratch_bytes < need) {
    set_error("scratch too small: need %zu bytes, got %zu", need, scratch_bytes);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  const Family fam = classify(desc);
  const KField F = make_field(desc);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* point_grads = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(scratch) + 255) & ~(uintptr_t)255);
  KCompositeBwd B{saved->weights,
                  saved->sample_density,
                  saved->sample_rgb,
                  saved->sample_semantics,
                  saved->accumulation,
                  up->d_rgb,
                  up->d_accumulation,
                  up->d_semantics,
                  up->d_weights,
                  up->d_sample_density,
                  up->d_sample_rgb,
                  up->d_sample_semantics,
                  point_grads,
                  desc->pass_semantic_gradients};
  if ((rc = launch_simt_composite_backward(Rr, B, st))) return rc;
  const bool tc = desc->impl != FNR_IMPL_SIMT;
  const KFieldBwd FB{point_grads, saved->stash_encoding};
  return launch_field_backward(fam, tc, F, P, G, Rr, FB, st);
}

int fnr_export_forward(const fnr_field_desc* desc, const fnr_field_params* params, const float* origins,
                       const float* normal, const float* bins, float near_plane, float far_plane, int32_t num_rays,
                       int32_t num_samples, uint64_t point_base, const fnr_export_params* xp, const fnr_export_out* out,
                       void* stream) {
  int rc = validate_desc(desc);
  if (rc) return rc;
  KParams P;
  if ((rc = make_params(desc, params, &P, "params"))) return rc;
  if (num_rays < 0 || num_samples < 1 || !xp || !out || !normal || !bins || (num_rays > 0 && !origins)) {
    set_error("invalid arguments to fnr_export_forward");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (!out->counts) {
    set_error("export counters are required");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  fnr_field_desc d2 = *desc;
  d2.position_mode = FNR_POS_AABB;    // setup_inference: field.spatial_distortion = None (fruit_nerf.py:183)
  d2.appearance_mode = FNR_APP_MEAN;  // get_inference_outputs (fruit_field.py:217-219)
  const KField F = make_field(&d2);
  KExport E;
  memset(&E, 0, sizeof(E));
  E.B = num_rays;
  E.S = num_samples;
  E.origins = origins;
  E.normal[0] = normal[0];
  E.normal[1] = normal[1];
  E.normal[2] = normal[2];
  E.bins = bins;
  if (xp->bins_ray_stride != 0 && xp->bins_ray_stride != num_samples + 1) {
    set_error("bins_ray_stride must be 0 (shared bins) or num_samples + 1 (per-ray bins), got %d", xp->bins_ray_stride);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  E.bins_ray_stride = xp->bins_ray_stride;
  E.near_plane = near_plane;
  E.far_plane = far_plane;
  E.logit_min = xp->semantic_logit_min;
  E.density_min = xp->density_min;
  E.label_thr = xp->label_sigmoid_threshold;
  E.capacity = xp->capacity;
  E.point_base = point_base;
  for (int k = 0; k < 3; ++k) {
    E.rows[k] = out->rows[k];
    E.keys[k] = out->keys[k];
  }
  E.counts = out->counts;
  E.sample_rgb = out->sample_rgb;
  E.point_location = out->point_location;
  E.sample_semantics = out->sample_semantics;
  E.sample_density = out->sample_density;
  E.semantics_colormap = out->semantics_colormap;
  const bool tc = desc->impl != FNR_IMPL_SIMT;
  return launch_export(classify(desc), tc, F, P, E, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_hash_indices(const fnr_field_desc* desc, const fnr_ray_batch* rays, int32_t* rows, float* positions, void* stream) {
  int rc = validate_desc(desc);
  if (rc) return rc;
  KRays Rr;
  fnr_field_desc d2 = *desc;
  d2.appearance_mode = FNR_APP_ZEROS;
  if ((rc = make_rays(&d2, rays, &Rr))) return rc;
  if (!rows) {
    set_error("rows is NULL");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  return launch_hash_indices(make_field(desc), Rr, rows, positions, reinterpret_cast<cudaStream_t>(stream));
}

static int make_density(const fnr_density_desc* d, const fnr_density_params* p, KDensity* K, const char* what) {
  if (!d || !p) {
    set_error("%s: NULL density desc/params", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  int max_levels, hidden, max_bins;
  proposal_limits(&max_levels, &hidden, &max_bins);
  if (d->num_levels < 1 || d->num_levels > max_levels || d->hidden_dim != hidden || d->log2_hashmap_size < 1 || d->log2_hashmap_size > 26) {
    set_error("unsupported proposal network (levels %d <= %d, hidden %d == %d)", d->num_levels, max_levels, d->hidden_dim, hidden);
    return FNR_ERR_UNSUPPORTED;
  }
  if (!p->hash_table || !p->w0 || !p->b0 || !p->w1 || !p->b1) {
    set_error("%s: NULL proposal parameter pointer", what);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  K->L = d->num_levels;
  K->log2T = d->log2_hashmap_size;
  K->position_mode = d->position_mode;
  memcpy(K->scalings, d->scalings, sizeof(K->scalings));
  memcpy(K->aabb, d->aabb, sizeof(K->aabb));
  K->hash_table = p->hash_table;
  K->w0 = p->w0;
  K->b0 = p->b0;
  K->w1 = p->w1;
  K->b1 = p->b1;
  return FNR_OK;
}

static int make_plain_rays(const fnr_ray_batch* r, KRays* K) {
  if (!r || r->num_rays < 0 || r->num_samples < 1 || (r->num_rays > 0 && (!r->origins || !r->directions || !r->starts || !r->ends))) {
    set_error("invalid ray batch");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  K->R = r->num_rays;
  K->S = r->num_samples;
  K->origins = r->origins;
  K->directions = r->directions;
  K->starts = r->starts;
  K->ends = r->ends;
  K->camera_indices = nullptr;
  return FNR_OK;
}

int fnr_proposal_weights_forward(const fnr_density_desc* desc, const fnr_density_params* params, const fnr_ray_batch* rays, float* density,
                                 float* weights, void* stream) {
  KDensity D;
  KRays Rr;
  int rc;
  if ((rc = make_density(desc, params, &D, "params"))) return rc;
  if ((rc = make_plain_rays(rays, &Rr))) return rc;
  if (!weights) {
    set_error("weights is NULL");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  return launch_proposal_weights_forward(D, Rr, density, weights, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_proposal_weights_backward(const fnr_density_desc* desc, const fnr_density_params* params, const fnr_ray_batch* rays,
                                  const float* density, const float* weights, const float* d_weights, const fnr_density_params* grads,
                                  void* stream) {
  KDensity D, G;
  KRays Rr;
  int rc;
  if ((rc = make_density(desc, params, &D, "params"))) return rc;
  if ((rc = make_density(desc, grads, &G, "grads"))) return rc;
  if ((rc = make_plain_rays(rays, &Rr))) return rc;
  if (!density || !weights || !d_weights) {
    set_error("density / weights / d_weights are required");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (Rr.S > 1024) {
    set_error("proposal backward supports at most 1024 samples per ray (got %d)", Rr.S);
    return FNR_ERR_UNSUPPORTED;
  }
  return launch_proposal_weights_backward(D, G, Rr, density, weights, d_weights, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_pdf_sample(const float* weights, const float* existing_bins, int32_t num_rays, int32_t num_existing, int32_t num_samples,
                   const float* u_base, const float* u_rand, int32_t u_stride, float anneal, const float* anneal_dev,
                   float histogram_padding, const float* nears, const float* fars, float* new_bins, float* starts, float* ends,
                   void* stream) {
  int max_levels, hidden, max_bins;
  proposal_limits(&max_levels, &hidden, &max_bins);
  if (num_rays < 0 || num_existing < 1 || num_samples < 1 || num_existing > max_bins || num_samples > max_bins) {
    set_error("pdf_sample: unsupported sizes (S=%d, num_samples=%d, max %d)", num_existing, num_samples, max_bins);
    return FNR_ERR_UNSUPPORTED;
  }
  if (num_rays > 0 && (!weights || !existing_bins || !u_base || !nears || !fars || !new_bins || !starts || !ends)) {
    set_error("pdf_sample: NULL argument");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  if (u_rand && u_stride != 1 && u_stride != num_samples + 1) {
    set_error("pdf_sample: u_stride must be 1 or num_samples+1");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KPdf A{num_rays, num_existing, num_samples, weights, existing_bins, u_base, u_rand, u_stride, anneal, histogram_padding, 1e-5f,
         anneal_dev, nears, fars, new_bins, starts, ends};
  return launch_pdf_sample(A, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_interlevel_loss(const float* c, const float* w, const float* cp, const float* wp, int32_t num_rays, int32_t sc, int32_t sp,
                        float mult, float* loss, float* d_wp, void* stream) {
  int max_levels, hidden, max_bins;
  proposal_limits(&max_levels, &hidden, &max_bins);
  if (num_rays < 0 || sc < 1 || sp < 1 || sp > max_bins) {
    set_error("interlevel_loss: unsupported sizes");
    return FNR_ERR_UNSUPPORTED;
  }
  if (num_rays > 0 && (!c || !w || !cp || !wp || !loss)) {
    set_error("interlevel_loss: NULL argument");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KInterlevel A{num_rays, sc, sp, c, w, cp, wp, num_rays > 0 ? mult / ((float)num_rays * (float)sc) : 0.f, loss, d_wp};
  return launch_interlevel_loss(A, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_adam_step(const fnr_adam_tensor* tensors, int32_t count, int32_t kind, const float* hyper, void* stream) {
  if (count < 0 || count > kMaxAdamTensors || (count > 0 && !tensors) || !hyper || (kind != FNR_OPT_ADAM && kind != FNR_OPT_RADAM)) {
    set_error("invalid arguments to fnr_adam_step (count %d, max %d)", count, kMaxAdamTensors);
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KAdam A;
  A.count = count;
  for (int i = 0; i < count; ++i) {
    const fnr_adam_tensor& t = tensors[i];
    if (t.n < 0 || (t.n > 0 && (!t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq))) {
      set_error("fnr_adam_step: tensor %d has NULL pointers", i);
      return FNR_ERR_INVALID_ARGUMENT;
    }
    A.t[i].param = t.param;
    A.t[i].grad = t.grad;
    A.t[i].exp_avg = t.exp_avg;
    A.t[i].exp_avg_sq = t.exp_avg_sq;
    A.t[i].n = t.n;
    const uintptr_t bits = reinterpret_cast<uintptr_t>(t.param) | reinterpret_cast<uintptr_t>(t.grad) |
                           reinterpret_cast<uintptr_t>(t.exp_avg) | reinterpret_cast<uintptr_t>(t.exp_avg_sq);
    A.t[i].vec4 = (bits & 15u) == 0;
  }
  return launch_adam(A, kind == FNR_OPT_RADAM, hyper, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_pixel_batch(const float* rand, const float* c2w, const float* images, const float* masks, int32_t num_images, int32_t height,
                    int32_t width, float fx, float fy, float cx, float cy, int32_t num_rays, float* origins, float* directions,
                    int32_t* camera_indices, int64_t* indices, float* image, float* fruit_mask, void* stream) {
  if (num_rays < 0 || num_images < 1 || height < 1 || width < 1 ||
      (num_rays > 0 && (!rand || !c2w || !images || !masks || !origins || !directions || !camera_indices || !image || !fruit_mask))) {
    set_error("invalid arguments to fnr_pixel_batch");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KPixelBatch A{num_rays, num_images, height, width, fx, fy, cx, cy, rand, c2w, images, masks, origins, directions, camera_indices, indices,
                image, fruit_mask};
  return launch_pixel_batch(A, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_spaced_bins(const float* base_bins, const float* t_rand, int32_t t_stride, const float* nears, const float* fars, int32_t num_rays,
                    int32_t num_samples, int32_t mode, float* bins, float* starts, float* ends, void* stream) {
  if (num_rays < 0 || num_samples < 1 || (mode != FNR_SPACING_UNIFORM && mode != FNR_SPACING_LINDISP_PIECEWISE) ||
      (t_rand && t_stride != 1 && t_stride != num_samples + 1) || (num_rays > 0 && (!base_bins || !nears || !fars || !bins || !starts || !ends))) {
    set_error("invalid arguments to fnr_spaced_bins");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KSpacedBins A{num_rays, num_samples, mode, base_bins, t_rand, t_stride, nears, fars, bins, starts, ends};
  return launch_spaced_bins(A, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_render_losses(const float* rgb, const float* semantics, const float* image, const float* fruit_mask, int32_t num_rays,
                      float semantic_weight, float* out, float* d_rgb, float* d_semantics, void* stream) {
  if (num_rays < 1 || !rgb || !semantics || !image || !fruit_mask || !out) {
    set_error("invalid arguments to fnr_render_losses");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KLosses A{num_rays, semantic_weight, rgb, semantics, image, fruit_mask, out, d_rgb, d_semantics};
  return launch_render_losses(A, reinterpret_cast<cudaStream_t>(stream));
}

int fnr_ray_metrics(const float* weights, const float* sdist, const float* starts, const float* ends, int32_t num_rays, int32_t num_samples,
                    float* distortion, float* median_depth, void* stream) {
  if (num_rays < 0 || num_samples < 1 || num_samples > 4096 || (num_rays > 0 && !weights) || (distortion && !sdist) ||
      (median_depth && (!starts || !ends))) {
    set_error("invalid arguments to fnr_ray_metrics");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  KRayMetrics A{num_rays, num_samples, weights, sdist, starts, ends, distortion, median_depth};
  return launch_ray_metrics(A, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
