"""ctypes binding of the C ABI declared in include/deepi2p_b200.h.

There is no CPU fallback: if the library is missing or a call fails, this raises.
"""
import ctypes
import os

from . import build as _build

_c = ctypes
_lib = None

EXPORTS = (
    "dib_abi_version", "dib_last_error", "dib_device_sm_count", "dib_profile_solve_events", "dib_evaluate_sliced", "frustum_solve_slice_after", "frustum_solve_slice_rounds",
    "frustum_solve_workspace_bytes", "frustum_solve_batch_f32", "frustum_solve_batch_f64", "frustum_solve_traced_f32",
    "frustum_register_workspace_bytes", "frustum_register_batch_f32",
    "frustum_evaluate_workspace_bytes",
    "frustum_evaluate_f32", "frustum_evaluate_f64", "frustum_residuals_f32", "frustum_residuals_f64",
    "frustum_poly_roots_f64", "frustum_interp_step_f64", "frustum_lm_next_step_f64",
    "frustum_prepare_workspace_bytes", "frustum_prepare_batch_f32", "frustum_sort_batch_f32",
    "frustum_inside_mask_f32", "pose_error_batch",
    "index_max_forward", "ball_query_forward", "ball_query_xyz_workspace_bytes", "ball_query_xyz_forward",
    "cluster_assign_workspace_bytes", "cluster_assign_forward",
    "pnp_ransac_workspace_bytes", "pnp_ransac_batch_f32", "epnp_batch_f64",
    "icp_workspace_bytes", "icp_register_batch_f32", "icp_register_batch_counted_f32", "icp_build_index_f32",
    "voxel_downsample_workspace_bytes", "voxel_downsample_batch_f32", "voxel_downsample_batch_f64",
    "estimate_normals_workspace_bytes",
    "estimate_normals_batch_f32", "nearest_batch_f32", "sym3_eig_batch_f64",
    "assemble_accumulate_workspace_bytes", "assemble_accumulate_f32",
    "assemble_accumulate_gather_workspace_bytes", "assemble_accumulate_gather_f32",
    "assemble_accumulate_f64_workspace_bytes", "assemble_accumulate_f64", "assemble_resample_workspace_bytes",
    "assemble_resample_f32", "assemble_candidates_workspace_bytes", "assemble_candidates_f32", "fps_batch_f32",
    "fps_batch_f64", "interp_weights_f32", "interp_forward_f32", "interp_backward_workspace_bytes",
    "interp_backward_f32", "image_assemble_workspace_bytes", "image_assemble_f32", "image_assemble_u8",
    "classifier_loss_workspace_bytes", "classifier_loss_forward_f32", "classifier_loss_backward_f32",
    "cluster_pool_forward_f32", "cluster_pool_backward_workspace_bytes", "cluster_pool_backward_f32",
    "knn_group_forward_f32", "knn_group_backward_workspace_bytes", "knn_group_backward_f32",
    "attn_fusion_forward_f32", "attn_fusion_backward_f32", "jpeg_decode_workspace_bytes", "jpeg_decode_batch_u8",
    "pointwise_mlp_packed_bytes", "pointwise_mlp_pack_f32", "pointwise_mlp_workspace_bytes", "pointwise_mlp_f32",
    "png_decode_workspace_bytes", "png_decode_batch_u8",
    "oxford_build_plan_f64", "oxford_build_count_workspace_bytes", "oxford_build_count_f64",
    "oxford_build_scatter_f64", "oxford_build_pack_f32",
    "oxford_debayer_workspace_bytes", "oxford_debayer_undistort_u8",
    "jpeg_encode_workspace_bytes", "jpeg_encode_entropy_u8", "jpeg_encode_stuff_u8",
    "knn_fusion_packed_bytes", "knn_fusion_pack_f32", "knn_fusion_f32", "pointwise_mlp_max_packed_bytes",
    "pointwise_mlp_max_pack_f32", "pointwise_mlp_max_workspace_bytes", "pointwise_mlp_max_f32",
    "node_mlp_packed_bytes", "node_mlp_pack_f32", "node_mlp_workspace_bytes", "node_mlp_f32",
)


EXPECTED_ABI = 4        # dib_abi_version() the argtypes below were written for


class NativeError(RuntimeError):
    pass


def lib_path():
    return _build.LIB


def load():
    """Load (building first if nvcc is available and the .so is stale/missing)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    override = os.environ.get("DIB_LIB_OVERRIDE")       # tuning aid: a prebuilt variant of the same library
    if override:
        if not os.path.exists(override):
            raise NativeError(f"DIB_LIB_OVERRIDE={override} does not exist")
        path = override
    elif not os.path.exists(path) or _build.is_stale():
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001 - turn any build problem into a loud, specific error
            if not os.path.exists(path):
                raise NativeError(
                    f"deepi2p_b200 CUDA library is missing ({path}) and could not be built: {e}. "
                    "There is no CPU fallback; run `python -m deepi2p_b200.build`.") from e
            import warnings
            warnings.warn(f"deepi2p_b200: {path} is older than its sources and the rebuild failed ({e}); "
                          "loading the stale library (its ABI version is checked)")
    lib = ctypes.CDLL(path)
    vp, i32, f64, sz = _c.c_void_p, _c.c_int, _c.c_double, _c.c_size_t
    lib.dib_abi_version.restype = i32
    abi = lib.dib_abi_version()
    if abi != EXPECTED_ABI:
        raise NativeError(f"{path} has ABI version {abi}, this binding was written for {EXPECTED_ABI}: "
                          "rebuild with `python -m deepi2p_b200.build --force`")
    lib.dib_last_error.restype = _c.c_char_p
    lib.dib_device_sm_count.restype = i32
    lib.dib_evaluate_sliced.restype = None
    lib.dib_evaluate_sliced.argtypes = [i32]
    lib.frustum_solve_slice_after.restype = i32
    lib.frustum_solve_slice_after.argtypes = [i32, i32, i32, i32]
    lib.frustum_solve_slice_rounds.restype = i32
    lib.frustum_solve_slice_rounds.argtypes = [i32, i32, i32, i32]
    lib.dib_profile_solve_events.restype = None
    lib.dib_profile_solve_events.argtypes = [vp, vp]
    lib.frustum_solve_workspace_bytes.restype = sz
    lib.frustum_solve_workspace_bytes.argtypes = [i32, i32, i32]
    lib.frustum_evaluate_workspace_bytes.restype = sz
    lib.frustum_evaluate_workspace_bytes.argtypes = [i32, i32]
    solve_args = [vp, vp, vp, i32, vp, vp, vp, vp, f64, f64, i32, i32, i32, i32,
                  vp, vp, vp, vp, vp, vp, vp, sz, vp]
    for name in ("frustum_solve_batch_f32", "frustum_solve_batch_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = solve_args
    lib.frustum_solve_traced_f32.restype = i32
    lib.frustum_solve_traced_f32.argtypes = solve_args[:20] + [vp, i32] + solve_args[20:]
    lib.frustum_register_workspace_bytes.restype = sz
    lib.frustum_register_workspace_bytes.argtypes = [i32, i32, i32]
    lib.frustum_register_batch_f32.restype = i32
    lib.frustum_register_batch_f32.argtypes = [vp, vp, i32, i32, i32, i32, _c.c_uint64, f64, f64, vp, vp, vp, f64, f64,
                                               i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    eval_args = [vp, vp, vp, i32, vp, vp, f64, f64, i32, i32, vp, vp, vp, vp, sz, vp]
    for name in ("frustum_evaluate_f32", "frustum_evaluate_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = eval_args
    res_args = [vp, vp, i32, i32, vp, vp, f64, f64, i32, vp, vp, vp]
    for name in ("frustum_residuals_f32", "frustum_residuals_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = res_args
    lib.frustum_poly_roots_f64.restype = i32
    lib.frustum_poly_roots_f64.argtypes = [vp, vp, i32, vp, vp]
    lib.frustum_interp_step_f64.restype = i32
    lib.frustum_interp_step_f64.argtypes = [vp, vp, i32, vp, vp]
    lib.frustum_lm_next_step_f64.restype = i32
    lib.frustum_lm_next_step_f64.argtypes = [i32, i32, vp, vp, vp, vp, vp]
    lib.frustum_prepare_workspace_bytes.restype = sz
    lib.frustum_prepare_workspace_bytes.argtypes = [i32, i32]
    lib.frustum_prepare_batch_f32.restype = i32
    lib.frustum_prepare_batch_f32.argtypes = [vp, vp, i32, i32, i32, i32, _c.c_uint64, f64, f64, i32,
                                              vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.frustum_sort_batch_f32.restype = i32
    lib.frustum_sort_batch_f32.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp]
    lib.frustum_inside_mask_f32.restype = i32
    lib.frustum_inside_mask_f32.argtypes = [vp, vp, i32, vp, vp, f64, f64, i32, vp, vp]
    lib.pose_error_batch.restype = i32
    lib.pose_error_batch.argtypes = [vp, vp, i32, f64, f64, vp, vp, vp, vp]
    lib.index_max_forward.restype = i32
    lib.index_max_forward.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp]
    lib.ball_query_xyz_workspace_bytes.restype = sz
    lib.ball_query_xyz_workspace_bytes.argtypes = [i32, i32]
    lib.ball_query_xyz_forward.restype = i32
    lib.ball_query_xyz_forward.argtypes = [vp, vp, _c.c_float, vp, i32, i32, i32, i32, vp, sz, vp]
    lib.cluster_assign_workspace_bytes.restype = sz
    lib.cluster_assign_workspace_bytes.argtypes = [i32, i32]
    lib.cluster_assign_forward.restype = i32
    lib.cluster_assign_forward.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.ball_query_forward.restype = i32
    lib.ball_query_forward.argtypes = [vp, _c.c_float, vp, i32, i32, i32, i32, vp]
    lib.pnp_ransac_workspace_bytes.restype = sz
    lib.pnp_ransac_workspace_bytes.argtypes = [i32, i32, i32]
    lib.pnp_ransac_batch_f32.restype = i32
    lib.pnp_ransac_batch_f32.argtypes = [vp, vp, vp, vp, i32, i32, vp, f64, f64, f64, i32, f64, f64, _c.c_uint64,
                                         vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.epnp_batch_f64.restype = i32
    lib.epnp_batch_f64.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp]
    lib.icp_workspace_bytes.restype = sz
    lib.icp_workspace_bytes.argtypes = [i32, i32, i32, i32]
    lib.icp_register_batch_f32.restype = i32
    lib.icp_register_batch_f32.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp, i32, f64, i32, f64, f64, i32,
                                           vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.icp_register_batch_counted_f32.restype = i32
    lib.icp_register_batch_counted_f32.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp, i32, f64, i32, f64, f64, i32,
                                                   vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.icp_build_index_f32.restype = i32
    lib.icp_build_index_f32.argtypes = [vp, vp, i32, i32, vp, sz, vp]
    lib.voxel_downsample_workspace_bytes.restype = sz
    lib.voxel_downsample_workspace_bytes.argtypes = [i32, i32, i32]
    for name in ("voxel_downsample_batch_f32", "voxel_downsample_batch_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i32, i32, vp, i32, f64, vp, vp, vp, vp, sz, vp]
    lib.estimate_normals_workspace_bytes.restype = sz
    lib.estimate_normals_workspace_bytes.argtypes = [i32, i32]
    lib.estimate_normals_batch_f32.restype = i32
    lib.estimate_normals_batch_f32.argtypes = [vp, vp, i32, i32, f64, i32, vp, vp, vp, vp, sz, vp]
    lib.nearest_batch_f32.restype = i32
    lib.nearest_batch_f32.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp, vp, sz, vp]
    lib.sym3_eig_batch_f64.restype = i32
    lib.sym3_eig_batch_f64.argtypes = [vp, i32, vp, vp, vp]
    lib.assemble_accumulate_workspace_bytes.restype = sz
    lib.assemble_accumulate_workspace_bytes.argtypes = [i32, i32, i32]
    lib.assemble_accumulate_f32.restype = i32
    lib.assemble_accumulate_f32.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, i32, f64, vp, vp, vp, i32, vp, vp, sz,
                                            vp]
    lib.assemble_accumulate_gather_workspace_bytes.restype = sz
    lib.assemble_accumulate_gather_workspace_bytes.argtypes = [i32, i32, i32]
    lib.assemble_accumulate_gather_f32.restype = i32
    lib.assemble_accumulate_gather_f32.argtypes = [vp, vp, vp, _c.c_int64, vp, vp, i32, i32, vp, vp, i32, f64, vp, vp,
                                                   vp, i32, vp, vp, sz, vp]
    lib.assemble_accumulate_f64_workspace_bytes.restype = sz
    lib.assemble_accumulate_f64_workspace_bytes.argtypes = [i32, i32, i32]
    lib.assemble_accumulate_f64.restype = i32
    lib.assemble_accumulate_f64.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, f64, vp, vp, vp, i32, vp, vp, sz, vp]
    lib.assemble_resample_workspace_bytes.restype = sz
    lib.assemble_resample_workspace_bytes.argtypes = [i32, i32]
    lib.assemble_resample_f32.restype = i32
    lib.assemble_resample_f32.argtypes = [vp, vp, vp, vp, i32, i32, i32, _c.c_uint64, vp, f64, f64, i32, vp, vp, vp,
                                          vp, vp, sz, vp]
    lib.assemble_candidates_workspace_bytes.restype = sz
    lib.assemble_candidates_workspace_bytes.argtypes = [i32, i32]
    lib.assemble_candidates_f32.restype = i32
    lib.assemble_candidates_f32.argtypes = [vp, i32, i32, _c.c_uint64, i32, i32, vp, vp, vp, sz, vp]
    for name in ("fps_batch_f32", "fps_batch_f64"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp]
    lib.interp_weights_f32.restype = i32
    lib.interp_weights_f32.argtypes = [vp, i32, vp, vp, i32, i32, i32, i32, vp, vp, vp]
    lib.interp_forward_f32.restype = i32
    lib.interp_forward_f32.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp]
    lib.interp_backward_workspace_bytes.restype = sz
    lib.interp_backward_workspace_bytes.argtypes = [i32, i32, i32, i32]
    lib.interp_backward_f32.restype = i32
    lib.interp_backward_f32.argtypes = [vp, _c.c_int64, vp, vp, i32, i32, i32, i32, i32, vp, vp, sz, vp]
    lib.image_assemble_workspace_bytes.restype = sz
    lib.image_assemble_workspace_bytes.argtypes = [i32, i32, i32]
    for name in ("image_assemble_f32", "image_assemble_u8"):
        getattr(lib, name).restype = i32
        getattr(lib, name).argtypes = [vp, sz, vp, vp, vp, i32, i32, i32, vp, vp, sz, vp]
    lib.classifier_loss_workspace_bytes.restype = sz
    lib.classifier_loss_workspace_bytes.argtypes = [i32, i32]
    lib.classifier_loss_forward_f32.restype = i32
    lib.classifier_loss_forward_f32.argtypes = [vp, _c.c_int64, vp, _c.c_int64, i32, vp, vp, vp, i32, i32, f64, f64,
                                                f64, i32, i32, f64, f64, i32, f64, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                                vp, vp, vp, vp, vp, sz, vp]
    lib.classifier_loss_backward_f32.restype = i32
    lib.classifier_loss_backward_f32.argtypes = [vp, _c.c_int64, vp, _c.c_int64, i32, i32, i32, vp, vp, vp, vp, vp, vp,
                                                 vp, f64, f64, i32, f64, vp, vp, vp]
    lib.cluster_pool_forward_f32.restype = i32
    lib.cluster_pool_forward_f32.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    lib.cluster_pool_backward_workspace_bytes.restype = sz
    lib.cluster_pool_backward_workspace_bytes.argtypes = [i32, i32, i32, i32]
    lib.cluster_pool_backward_f32.restype = i32
    lib.cluster_pool_backward_f32.argtypes = [vp, vp, _c.c_int64, vp, vp, vp, i32, i32, i32, i32, vp, vp, sz, vp]
    lib.knn_group_forward_f32.restype = i32
    lib.knn_group_forward_f32.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]
    lib.knn_group_backward_workspace_bytes.restype = sz
    lib.knn_group_backward_workspace_bytes.argtypes = [i32, i32, i32, i32, i32]
    lib.knn_group_backward_f32.restype = i32
    lib.knn_group_backward_f32.argtypes = [vp, _c.c_int64, vp, i32, i32, i32, i32, i32, vp, vp, sz, vp]
    lib.attn_fusion_forward_f32.restype = i32
    lib.attn_fusion_forward_f32.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp]
    lib.attn_fusion_backward_f32.restype = i32
    lib.attn_fusion_backward_f32.argtypes = [vp, _c.c_int64, vp, vp, i32, i32, i32, i32, vp, vp, vp]
    lib.jpeg_decode_workspace_bytes.restype = sz
    lib.jpeg_decode_workspace_bytes.argtypes = [vp, i32, sz, i32]
    lib.jpeg_decode_batch_u8.restype = i32
    lib.jpeg_decode_batch_u8.argtypes = [vp, sz, vp, vp, vp, i32, i32, vp, sz, vp, vp, sz, vp]
    lib.pointwise_mlp_packed_bytes.restype = sz
    lib.pointwise_mlp_packed_bytes.argtypes = [vp, i32, vp, i32]
    lib.pointwise_mlp_pack_f32.restype = i32
    lib.pointwise_mlp_pack_f32.argtypes = [vp, i32, vp, i32, vp, sz, vp]
    lib.pointwise_mlp_workspace_bytes.restype = sz
    lib.pointwise_mlp_workspace_bytes.argtypes = [vp, i32, vp, i32, i32]
    lib.pointwise_mlp_f32.restype = i32
    lib.pointwise_mlp_f32.argtypes = [vp, i32, vp, i32, vp, sz, i32, i32, i32, vp, vp, vp, vp, sz, vp]
    lib.knn_fusion_packed_bytes.restype = sz
    lib.knn_fusion_packed_bytes.argtypes = [i32, vp, i32, i32]
    lib.knn_fusion_pack_f32.restype = i32
    lib.knn_fusion_pack_f32.argtypes = [i32, vp, i32, i32, vp, sz, vp]
    lib.knn_fusion_f32.restype = i32
    lib.knn_fusion_f32.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp, i32, i32, vp, sz, vp, vp, vp]
    lib.pointwise_mlp_max_packed_bytes.restype = sz
    lib.pointwise_mlp_max_packed_bytes.argtypes = [i32, vp, i32]
    lib.pointwise_mlp_max_pack_f32.restype = i32
    lib.pointwise_mlp_max_pack_f32.argtypes = [i32, vp, i32, vp, sz, vp]
    lib.pointwise_mlp_max_workspace_bytes.restype = sz
    lib.pointwise_mlp_max_workspace_bytes.argtypes = [i32, i32, i32]
    lib.pointwise_mlp_max_f32.restype = i32
    lib.pointwise_mlp_max_f32.argtypes = [vp, i32, vp, i32, vp, sz, i32, i32, vp, vp, sz, vp]
    lib.node_mlp_packed_bytes.restype = sz
    lib.node_mlp_packed_bytes.argtypes = [vp, i32, vp, i32]
    lib.node_mlp_pack_f32.restype = i32
    lib.node_mlp_pack_f32.argtypes = [vp, i32, vp, i32, vp, sz, vp]
    lib.node_mlp_workspace_bytes.restype = sz
    lib.node_mlp_workspace_bytes.argtypes = [vp, i32, vp, i32, i32]
    lib.node_mlp_f32.restype = i32
    lib.node_mlp_f32.argtypes = [vp, i32, vp, i32, vp, sz, i32, i32, vp, vp, sz, vp]
    lib.png_decode_workspace_bytes.restype = sz
    lib.png_decode_workspace_bytes.argtypes = [vp, i32, vp, i32, sz]
    lib.png_decode_batch_u8.restype = i32
    lib.png_decode_batch_u8.argtypes = [vp, sz, vp, i32, vp, i32, vp, sz, vp, vp, sz, vp]
    i64 = _c.c_int64
    lib.oxford_build_plan_f64.restype = i32
    lib.oxford_build_plan_f64.argtypes = [vp, vp, i64, vp, vp, i32, vp, f64, i32, vp, vp, vp, vp, vp]
    lib.oxford_build_count_workspace_bytes.restype = sz
    lib.oxford_build_count_workspace_bytes.argtypes = [i32, i32]
    lib.oxford_build_count_f64.restype = i32
    lib.oxford_build_count_f64.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, f64, vp, vp, vp, vp, sz, vp]
    lib.oxford_build_scatter_f64.restype = i32
    lib.oxford_build_scatter_f64.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, f64, i32, vp, vp, vp]
    lib.oxford_build_pack_f32.restype = i32
    lib.oxford_build_pack_f32.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, vp, vp]
    lib.oxford_debayer_workspace_bytes.restype = sz
    lib.oxford_debayer_workspace_bytes.argtypes = [i32]
    lib.oxford_debayer_undistort_u8.restype = i32
    lib.oxford_debayer_undistort_u8.argtypes = [vp, sz, vp, i64, vp, i32, vp, sz, vp, sz, vp]
    lib.jpeg_encode_workspace_bytes.restype = sz
    lib.jpeg_encode_workspace_bytes.argtypes = [vp, i32]
    lib.jpeg_encode_entropy_u8.restype = i32
    lib.jpeg_encode_entropy_u8.argtypes = [vp, sz, vp, i32, vp, vp, vp, vp, sz, vp]
    lib.jpeg_encode_stuff_u8.restype = i32
    lib.jpeg_encode_stuff_u8.argtypes = [vp, i32, vp, vp, sz, vp, sz, vp]
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().dib_last_error().decode("utf-8", "replace")
        raise NativeError(f"{what} failed (code {rc}): {msg}")
