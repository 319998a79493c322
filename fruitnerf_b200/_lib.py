"""ctypes binding of libfruitnerf_b200.so (the C ABI of include/fruitnerf_b200.h).

There is no CPU or PyTorch fallback: if the library is missing, loading raises, and every op in
``fruitnerf_b200.ops`` requires CUDA tensors.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

ABI_VERSION = 2  # FNR_ABI_VERSION of include/fruitnerf_b200.h
FNR_MAX_LEVELS = 32
FNR_MAX_LAYERS = 4

FNR_POS_CONTRACT, FNR_POS_AABB = 0, 1
FNR_APP_PER_CAMERA, FNR_APP_MEAN, FNR_APP_ZEROS = 0, 1, 2
FNR_IMPL_AUTO, FNR_IMPL_SIMT, FNR_IMPL_TCGEN05 = 0, 1, 2
FNR_SPACING_UNIFORM, FNR_SPACING_LINDISP_PIECEWISE = 0, 1

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u64p = C.POINTER(C.c_uint64)


class MlpDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("dims", C.c_int32 * (FNR_MAX_LAYERS + 1))]


class FieldDesc(C.Structure):
    _fields_ = [
        ("num_levels", C.c_int32),
        ("features_per_level", C.c_int32),
        ("log2_hashmap_size", C.c_int32),
        ("scalings", C.c_float * FNR_MAX_LEVELS),
        ("geo_feat_dim", C.c_int32),
        ("appearance_dim", C.c_int32),
        ("num_images", C.c_int32),
        ("base", MlpDesc),
        ("semantic", MlpDesc),
        ("color", MlpDesc),
        ("aabb", C.c_float * 6),
        ("position_mode", C.c_int32),
        ("appearance_mode", C.c_int32),
        ("pass_semantic_gradients", C.c_int32),
        ("impl", C.c_int32),
    ]


class FieldParams(C.Structure):
    _fields_ = [
        ("hash_table", C.c_void_p),
        ("base_w", C.c_void_p * FNR_MAX_LAYERS),
        ("base_b", C.c_void_p * FNR_MAX_LAYERS),
        ("sem_w", C.c_void_p * FNR_MAX_LAYERS),
        ("sem_b", C.c_void_p * FNR_MAX_LAYERS),
        ("head_w", C.c_void_p),
        ("head_b", C.c_void_p),
        ("col_w", C.c_void_p * FNR_MAX_LAYERS),
        ("col_b", C.c_void_p * FNR_MAX_LAYERS),
        ("app_embedding", C.c_void_p),
    ]


class RayBatch(C.Structure):
    _fields_ = [
        ("num_rays", C.c_int32),
        ("num_samples", C.c_int32),
        ("origins", C.c_void_p),
        ("directions", C.c_void_p),
        ("starts", C.c_void_p),
        ("ends", C.c_void_p),
        ("camera_indices", C.c_void_p),
    ]


class RenderOut(C.Structure):
    _fields_ = [
        ("rgb", C.c_void_p),
        ("accumulation", C.c_void_p),
        ("depth", C.c_void_p),
        ("depth_index", C.c_void_p),
        ("semantics", C.c_void_p),
        ("weights", C.c_void_p),
        ("sample_density", C.c_void_p),
        ("sample_rgb", C.c_void_p),
        ("sample_semantics", C.c_void_p),
        ("stash_encoding", C.c_void_p),
        ("clamp_rgb", C.c_int32),
    ]


class RenderGrads(C.Structure):
    _fields_ = [
        ("d_rgb", C.c_void_p),
        ("d_accumulation", C.c_void_p),
        ("d_semantics", C.c_void_p),
        ("d_weights", C.c_void_p),
        ("d_sample_density", C.c_void_p),
        ("d_sample_rgb", C.c_void_p),
        ("d_sample_semantics", C.c_void_p),
    ]


class RenderSaved(C.Structure):
    _fields_ = [
        ("weights", C.c_void_p),
        ("sample_density", C.c_void_p),
        ("sample_rgb", C.c_void_p),
        ("sample_semantics", C.c_void_p),
        ("stash_encoding", C.c_void_p),
        ("accumulation", C.c_void_p),
    ]


class ExportParams(C.Structure):
    _fields_ = [
        ("semantic_logit_min", C.c_float),
        ("density_min", C.c_float),
        ("label_sigmoid_threshold", C.c_float),
        ("capacity", C.c_int32),
        ("bins_ray_stride", C.c_int32),
    ]


class NvlsDesc(C.Structure):
    _fields_ = [
        ("multicast_ptr", C.c_void_p),
        ("local_ptr", C.c_void_p),
        ("multicast_bf16", C.c_void_p),
        ("local_bf16", C.c_void_p),
        ("signal_pads", C.c_void_p),
        ("grid_counter", C.c_void_p),
        ("rank", C.c_int32),
        ("world_size", C.c_int32),
        ("signal_slots", C.c_int32),
        ("signal_slot_base", C.c_int32),
    ]


class ExportOut(C.Structure):
    _fields_ = [
        ("rows", C.c_void_p * 3),
        ("keys", C.c_void_p * 3),
        ("counts", C.c_void_p),
        ("sample_rgb", C.c_void_p),
        ("point_location", C.c_void_p),
        ("sample_semantics", C.c_void_p),
        ("sample_density", C.c_void_p),
        ("semantics_colormap", C.c_void_p),
    ]


class DensityDesc(C.Structure):
    _fields_ = [
        ("num_levels", C.c_int32),
        ("log2_hashmap_size", C.c_int32),
        ("hidden_dim", C.c_int32),
        ("scalings", C.c_float * FNR_MAX_LEVELS),
        ("aabb", C.c_float * 6),
        ("position_mode", C.c_int32),
    ]


class DensityParams(C.Structure):
    _fields_ = [("hash_table", C.c_void_p), ("w0", C.c_void_p), ("b0", C.c_void_p), ("w1", C.c_void_p), ("b1", C.c_void_p)]


class AdamTensor(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("n", C.c_int64)]


class FrameOutput(C.Structure):
    _fields_ = [("image", C.c_void_p), ("kind", C.c_int32), ("auto_range", C.c_int32), ("near_plane", C.c_double),
                ("far_plane", C.c_double)]


FNR_CAMERA_PERSPECTIVE, FNR_CAMERA_FISHEYE, FNR_CAMERA_EQUIRECTANGULAR = 0, 1, 2
FNR_FRAME_COLOR, FNR_FRAME_TURBO, FNR_FRAME_DEPTH = 0, 1, 2
FNR_RANGE_AUTO_NEAR, FNR_RANGE_AUTO_FAR = 1, 2
FNR_MAX_FRAME_OUTPUTS = 8
FNR_COMPOSE_SCRATCH_FLOATS = FNR_MAX_FRAME_OUTPUTS * 256 * 2

FNR_OPT_ADAM, FNR_OPT_RADAM = 0, 1
FNR_MESH_ASSIGN_SCRATCH_BYTES = 256
FNR_MAX_ADAM_TENSORS = 48
FNR_IMAGE_RECORD_DOUBLES = 12
FNR_TEXTURE_MAX_SIDE = 16384
FNR_MEAN_EDGE_DOUBLES = 1 + 256
FNR_UNWRAP_MIN_SIDE = 16
FNR_UNWRAP_MARGIN = 3
FNR_UNWRAP_GUTTER = 2
FNR_UNWRAP_BISECTIONS = 40
FNR_UNWRAP_STAGES = 5
# record slots of fnr_image_stats / fnr_ssim (FNR_REC_* of the header), in order
IMAGE_RECORD_FIELDS = ("sse", "rgb_min", "rgb_max", "image_min", "image_max", "accumulation_sum", "fruit_tp", "fruit_fp", "fruit_fn",
                       "fruit_tn", "ssim", "data_range")

LIB_PATH = Path(__file__).resolve().parent / "csrc" / "libfruitnerf_b200.so"

# every symbol include/fruitnerf_b200.h declares
EXPORTED_SYMBOLS = (
    "fnr_version",
    "fnr_launch_count",
    "fnr_nvls_allreduce_mean",
    "fnr_last_error",
    "fnr_render_forward",
    "fnr_render_backward",
    "fnr_render_backward_scratch_bytes",
    "fnr_export_forward",
    "fnr_hash_indices",
    "fnr_level_scatter",
    "fnr_proposal_weights_forward",
    "fnr_proposal_weights_backward",
    "fnr_pdf_sample",
    "fnr_interlevel_loss",
    "fnr_adam_step",
    "fnr_pixel_batch",
    "fnr_spaced_bins",
    "fnr_render_losses",
    "fnr_ray_metrics",
    "fnr_cluster_scratch_bytes",
    "fnr_radius_count",
    "fnr_voxel_down_sample",
    "fnr_dbscan",
    "fnr_radius_count_multi",
    "fnr_cluster_sums",
    "fnr_knn_mean_distance",
    "fnr_estimate_normals",
    "fnr_backproject_select",
    "fnr_icp_scaled",
    "fnr_ward_cut",
    "fnr_hausdorff",
    "fnr_camera_rays",
    "fnr_compose_frame",
    "fnr_pixel_batch_lens",
    "fnr_camera_rays_lens",
    "fnr_tsdf_integrate",
    "fnr_marching_cubes_scratch_bytes",
    "fnr_marching_cubes_count",
    "fnr_marching_cubes_emit",
    "fnr_poisson_scratch_bytes",
    "fnr_poisson_splat",
    "fnr_poisson_apply",
    "fnr_poisson_solve",
    "fnr_poisson_sample",
    "fnr_mesh_measure_scratch_bytes",
    "fnr_mesh_components",
    "fnr_mesh_assign_centers",
    "fnr_mesh_measure_groups",
    "fnr_image_metrics_scratch_bytes",
    "fnr_image_stats",
    "fnr_ssim",
    "fnr_texture_atlas_size",
    "fnr_texel_rays",
    "fnr_mesh_mean_edge",
    "fnr_mesh_decimate_scratch_bytes",
    "fnr_mesh_decimate",
    "fnr_chart_unwrap_scratch_bytes",
    "fnr_chart_unwrap",
    "fnr_chart_texel_rays",
)

_lib = None


class FruitNerfNativeError(RuntimeError):
    pass


def load() -> C.CDLL:
    """dlopen the C-ABI library.  Raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise FruitNerfNativeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  fruitnerf_b200 has no CPU / PyTorch fallback."
        )
    lib = C.CDLL(str(LIB_PATH))
    lib.fnr_version.restype = C.c_int
    lib.fnr_nvls_allreduce_mean.restype = C.c_int
    lib.fnr_nvls_allreduce_mean.argtypes = [C.POINTER(NvlsDesc), C.c_size_t, C.c_int32, C.c_void_p]
    lib.fnr_launch_count.restype = C.c_uint64
    lib.fnr_launch_count.argtypes = [C.c_int32]
    lib.fnr_last_error.restype = C.c_char_p
    lib.fnr_render_forward.restype = C.c_int
    lib.fnr_render_forward.argtypes = [C.POINTER(FieldDesc), C.POINTER(FieldParams), C.POINTER(RayBatch), C.POINTER(RenderOut), C.c_void_p]
    lib.fnr_render_backward.restype = C.c_int
    lib.fnr_render_backward.argtypes = [
        C.POINTER(FieldDesc), C.POINTER(FieldParams), C.POINTER(RayBatch), C.POINTER(RenderSaved),
        C.POINTER(RenderGrads), C.POINTER(FieldParams), C.c_void_p, C.c_size_t, C.c_void_p,
    ]
    lib.fnr_render_backward_scratch_bytes.restype = C.c_int
    lib.fnr_render_backward_scratch_bytes.argtypes = [C.POINTER(FieldDesc), C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]
    lib.fnr_export_forward.restype = C.c_int
    lib.fnr_export_forward.argtypes = [
        C.POINTER(FieldDesc), C.POINTER(FieldParams), C.c_void_p, _f32p, C.c_void_p, C.c_float, C.c_float,
        C.c_int32, C.c_int32, C.c_uint64, C.POINTER(ExportParams), C.POINTER(ExportOut), C.c_void_p,
    ]
    lib.fnr_hash_indices.restype = C.c_int
    lib.fnr_hash_indices.argtypes = [C.POINTER(FieldDesc), C.POINTER(RayBatch), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fnr_level_scatter.restype = C.c_int
    lib.fnr_level_scatter.argtypes = [C.POINTER(FieldDesc), C.POINTER(RayBatch), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fnr_proposal_weights_forward.restype = C.c_int
    lib.fnr_proposal_weights_forward.argtypes = [C.POINTER(DensityDesc), C.POINTER(DensityParams), C.POINTER(RayBatch), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fnr_proposal_weights_backward.restype = C.c_int
    lib.fnr_proposal_weights_backward.argtypes = [C.POINTER(DensityDesc), C.POINTER(DensityParams), C.POINTER(RayBatch), C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.POINTER(DensityParams), C.c_void_p]
    lib.fnr_pdf_sample.restype = C.c_int
    lib.fnr_pdf_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_float,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fnr_interlevel_loss.restype = C.c_int
    lib.fnr_interlevel_loss.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
    lib.fnr_adam_step.restype = C.c_int
    lib.fnr_adam_step.argtypes = [C.POINTER(AdamTensor), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    vp, i32, f32 = C.c_void_p, C.c_int32, C.c_float
    lib.fnr_pixel_batch.restype = C.c_int
    lib.fnr_pixel_batch.argtypes = [vp, vp, vp, vp, i32, i32, i32, f32, f32, f32, f32, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.fnr_spaced_bins.restype = C.c_int
    lib.fnr_spaced_bins.argtypes = [vp, vp, i32, vp, vp, i32, i32, i32, vp, vp, vp, vp]
    lib.fnr_render_losses.restype = C.c_int
    lib.fnr_render_losses.argtypes = [vp, vp, vp, vp, i32, f32, vp, vp, vp, vp]
    lib.fnr_ray_metrics.restype = C.c_int
    lib.fnr_ray_metrics.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp]
    i64, f64, f64p, sz = C.c_int64, C.c_double, C.POINTER(C.c_double), C.c_size_t
    lib.fnr_cluster_scratch_bytes.restype = C.c_int
    lib.fnr_cluster_scratch_bytes.argtypes = [i64, C.POINTER(C.c_size_t)]
    lib.fnr_radius_count.restype = C.c_int
    lib.fnr_radius_count.argtypes = [vp, i64, f64p, f64p, f64, i32, vp, vp, sz, vp]
    lib.fnr_voxel_down_sample.restype = C.c_int
    lib.fnr_voxel_down_sample.argtypes = [vp, i64, f64p, f64p, f64, vp, vp, vp, sz, vp]
    lib.fnr_dbscan.restype = C.c_int
    lib.fnr_dbscan.argtypes = [vp, i64, f64p, f64p, f64, i32, vp, vp, vp, sz, vp]
    i32p = C.POINTER(C.c_int32)
    lib.fnr_radius_count_multi.restype = C.c_int
    lib.fnr_radius_count_multi.argtypes = [vp, i64, f64p, f64p, f64p, i32p, i32, vp, vp, sz, vp]
    lib.fnr_cluster_sums.restype = C.c_int
    lib.fnr_cluster_sums.argtypes = [vp, vp, i64, i32, vp, vp, vp, sz, vp]
    lib.fnr_knn_mean_distance.restype = C.c_int
    lib.fnr_knn_mean_distance.argtypes = [vp, i64, f64p, f64p, i32, vp, vp, sz, vp]
    lib.fnr_estimate_normals.restype = C.c_int
    lib.fnr_estimate_normals.argtypes = [vp, i64, f64p, f64p, i32, vp, vp, vp, sz, vp]
    lib.fnr_backproject_select.restype = C.c_int
    lib.fnr_backproject_select.argtypes = [vp, vp, vp, vp, vp, i32, i32, _f32p, _f32p, i32, vp, vp, vp, vp, vp]
    lib.fnr_icp_scaled.restype = C.c_int
    lib.fnr_icp_scaled.argtypes = [vp, i32, vp, vp, i32, i32, vp, f64, i32, f64, f64, vp, vp, vp, vp, vp]
    lib.fnr_ward_cut.restype = C.c_int
    lib.fnr_ward_cut.argtypes = [vp, vp, i32, i32, vp, vp]
    lib.fnr_hausdorff.restype = C.c_int
    lib.fnr_hausdorff.argtypes = [vp, vp, vp, vp, i32, vp, vp]
    lib.fnr_camera_rays.restype = C.c_int
    lib.fnr_camera_rays.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i64, i32, vp, vp, vp]
    lib.fnr_compose_frame.restype = C.c_int
    lib.fnr_compose_frame.argtypes = [C.POINTER(FrameOutput), i32, vp, i32, i32, vp, vp, vp, vp]
    lib.fnr_pixel_batch_lens.restype = C.c_int
    lib.fnr_pixel_batch_lens.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.fnr_camera_rays_lens.restype = C.c_int
    lib.fnr_camera_rays_lens.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i64, i32, vp, vp, vp]
    lib.fnr_tsdf_integrate.restype = C.c_int
    lib.fnr_tsdf_integrate.argtypes = [vp, vp, vp, vp, i64, i64, i64, _f32p, _f32p, f32, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, vp]
    lib.fnr_marching_cubes_scratch_bytes.restype = C.c_int
    lib.fnr_marching_cubes_scratch_bytes.argtypes = [i64, i64, i64, C.POINTER(C.c_size_t)]
    lib.fnr_marching_cubes_count.restype = C.c_int
    lib.fnr_marching_cubes_count.argtypes = [vp, i64, i64, i64, vp, sz, vp, vp]
    lib.fnr_marching_cubes_emit.restype = C.c_int
    lib.fnr_marching_cubes_emit.argtypes = [vp, vp, vp, i64, i64, i64, _f32p, _f32p, vp, sz, i64, i64, vp, vp, vp, vp, vp, vp]
    lib.fnr_poisson_scratch_bytes.restype = C.c_int
    lib.fnr_poisson_scratch_bytes.argtypes = [i64, i32, C.POINTER(C.c_size_t)]
    lib.fnr_poisson_splat.restype = C.c_int
    lib.fnr_poisson_splat.argtypes = [vp, vp, vp, vp, i64, i32, f64p, f64, vp, sz, vp, vp, vp, vp, vp, vp]
    lib.fnr_poisson_apply.restype = C.c_int
    lib.fnr_poisson_apply.argtypes = [i64, i32, f32, vp, sz, vp, vp, vp]
    lib.fnr_poisson_solve.restype = C.c_int
    lib.fnr_poisson_solve.argtypes = [vp, vp, vp, vp, i64, i32, f64p, f64, f32, i32, f32, vp, sz, vp, vp, vp, vp, _i64p, f64p, vp]
    lib.fnr_poisson_sample.restype = C.c_int
    lib.fnr_poisson_sample.argtypes = [vp, i64, i32, f64p, f64, vp, vp, vp]
    lib.fnr_mesh_measure_scratch_bytes.restype = C.c_int
    lib.fnr_mesh_measure_scratch_bytes.argtypes = [i64, i64, C.POINTER(C.c_size_t)]
    lib.fnr_mesh_components.restype = C.c_int
    lib.fnr_mesh_components.argtypes = [vp, i64, i64, vp, sz, vp, _i64p, vp]
    lib.fnr_mesh_assign_centers.restype = C.c_int
    lib.fnr_mesh_assign_centers.argtypes = [vp, vp, i64, i64, vp, i64, f64, vp, sz, vp, vp]
    lib.fnr_mesh_measure_groups.restype = C.c_int
    lib.fnr_mesh_measure_groups.argtypes = [vp, vp, i64, i64, vp, i64, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.fnr_image_metrics_scratch_bytes.restype = C.c_int
    lib.fnr_image_metrics_scratch_bytes.argtypes = [i32, i32, C.POINTER(C.c_size_t)]
    lib.fnr_image_stats.restype = C.c_int
    lib.fnr_image_stats.argtypes = [vp, vp, vp, vp, vp, i32, i32, vp, sz, vp, vp]
    lib.fnr_ssim.restype = C.c_int
    lib.fnr_ssim.argtypes = [vp, vp, i32, i32, vp, sz, vp, vp]
    lib.fnr_texture_atlas_size.restype = C.c_int
    lib.fnr_texture_atlas_size.argtypes = [i64, i32, _i64p, _i64p]
    lib.fnr_texel_rays.restype = C.c_int
    lib.fnr_texel_rays.argtypes = [vp, vp, vp, i64, i32, i32, i32, f32, i64, i32, vp, vp, vp]
    lib.fnr_mesh_mean_edge.restype = C.c_int
    lib.fnr_mesh_mean_edge.argtypes = [vp, vp, i64, vp, vp]
    lib.fnr_mesh_decimate_scratch_bytes.restype = C.c_int
    lib.fnr_mesh_decimate_scratch_bytes.argtypes = [i64, i64, C.POINTER(C.c_size_t)]
    lib.fnr_mesh_decimate.restype = C.c_int
    lib.fnr_mesh_decimate.argtypes = [vp, vp, i64, i64, i64, vp, sz, vp, vp, vp, _i64p, _i64p, C.POINTER(C.c_int32), vp]
    lib.fnr_chart_unwrap_scratch_bytes.restype = C.c_int
    lib.fnr_chart_unwrap_scratch_bytes.argtypes = [i64, i64, i32, C.POINTER(C.c_size_t)]
    lib.fnr_chart_unwrap.restype = C.c_int
    lib.fnr_chart_unwrap.argtypes = [vp, vp, i64, i64, i32, vp, sz, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int32), _i64p, f64p, _i64p,
                                     f64p, vp]
    lib.fnr_chart_texel_rays.restype = C.c_int
    lib.fnr_chart_texel_rays.argtypes = [vp, vp, vp, i64, vp, vp, i64, f32, i64, i32, vp, vp, vp]
    if lib.fnr_version() != ABI_VERSION:
        raise FruitNerfNativeError(f"ABI version mismatch: library reports {lib.fnr_version()}")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().fnr_last_error().decode("utf-8", "replace")
        if rc == -1 and "Camera indices are not provided" in msg:
            raise AttributeError(msg)  # fruit_field.py:240-241
        raise FruitNerfNativeError(f"fruitnerf_b200 native call failed (code {rc}): {msg}")
