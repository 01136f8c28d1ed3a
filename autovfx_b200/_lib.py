"""ctypes binding of the C-ABI library (include/gsr_b200.h).

There is NO fallback: if libgsr_b200.so cannot be loaded (and cannot be built because nvcc is absent)
importing this module raises, and every operator of the package fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.utils.deterministic

from . import build as _build

_f32p = C.c_void_p  # device pointers travel as plain integers


class gsr_frame(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("D", C.c_int32), ("M", C.c_int32), ("W", C.c_int32), ("H", C.c_int32),
        ("scale_modifier", C.c_float), ("tanfovx", C.c_float), ("tanfovy", C.c_float),
        ("prefiltered", C.c_int32), ("debug", C.c_int32),
        ("bg", _f32p), ("means3D", _f32p), ("shs", _f32p), ("colors_precomp", _f32p), ("opacities", _f32p),
        ("scales", _f32p), ("rotations", _f32p), ("cov3D_precomp", _f32p), ("viewmatrix", _f32p),
        ("projmatrix", _f32p), ("campos", _f32p),
    ]


class gsr_workspace(C.Structure):
    _fields_ = [("geom", C.c_void_p), ("geom_bytes", C.c_size_t), ("binning", C.c_void_p), ("binning_bytes", C.c_size_t),
                ("image", C.c_void_p), ("image_bytes", C.c_size_t)]


class gsr_counters(C.Structure):
    _fields_ = [("num_rendered", C.c_uint32), ("overflow", C.c_uint32), ("max_tile", C.c_uint32), ("trapped", C.c_uint32),
                ("num_visible", C.c_uint32), ("foot_total", C.c_uint32), ("exact_redos", C.c_uint32),
                ("reserved", C.c_uint32)]


class gsr_grads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_ddepths", "dL_dmeans3D",
                                          "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations")]


class gsr_views(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("records", "cov3D", "clamped", "point_list", "sorted_keys", "ranges", "n_contrib",
                                          "tile_count", "tile_big", "counters")]


class gsr_object_xform(C.Structure):
    _fields_ = [("rotation", C.c_float * 9), ("quat", C.c_float * 4), ("center", C.c_float * 3), ("initial_center", C.c_float * 3),
                ("scaling", C.c_float), ("log_scaling", C.c_float)]


class gsr_densify_group(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("m1_src", C.c_void_p), ("m1_dst", C.c_void_p), ("m2_src", C.c_void_p),
                ("m2_dst", C.c_void_p), ("width", C.c_int32), ("role", C.c_int32)]


class gsr_adam_tensor(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("numel", C.c_int64),
                ("lerp_weight", C.c_float), ("beta2", C.c_float), ("one_minus_beta2", C.c_float), ("bias_correction2_sqrt", C.c_float),
                ("eps", C.c_float), ("step_size", C.c_float)]


class gsr_png_image(C.Structure):
    _fields_ = [("data", C.c_void_p), ("stride_h", C.c_int64), ("stride_w", C.c_int64), ("stride_c", C.c_int64), ("H", C.c_int32),
                ("W", C.c_int32), ("C", C.c_int32), ("flags", C.c_int32), ("lut", C.c_void_p)]


GSR_PNG_SWAP_RB = 1
GSR_PNG_MAX_BATCH = 16
GSR_ADAM_MAX_TENSORS = 32
GSR_LOSS_REDUCE_BYTES = 256 + 16 * 1024
GSR_DENSIFY_MAX_GROUPS = 8
GSR_DENSIFY_ROLE_COPY, GSR_DENSIFY_ROLE_XYZ, GSR_DENSIFY_ROLE_SCALING = 0, 1, 2
GSR_DENSIFY_ROTATION_3DGS, GSR_DENSIFY_ROTATION_SUGAR = 0, 1
GSR_FLAG_FOR_BACKWARD = 1
GSR_FLAG_SORTED_KEYS = 2
GSR_FLAG_TIGHT_TILES = 4
GSR_FLAG_REUSE_GEOMETRY = 8
GSR_FLAG_EXACT_IMAGES = 16
GSR_FLAG_BINNING_ONLY = 32
GSR_FLAG_RESUME = 64
GSR_SLAB_SHIFT = 16
ABI_VERSION = 4

_int, _i32, _i64, _f32, _size, _ptr = C.c_int, C.c_int32, C.c_int64, C.c_float, C.c_size_t, C.c_void_p
_frame, _ws, _grads = C.POINTER(gsr_frame), C.POINTER(gsr_workspace), C.POINTER(gsr_grads)
_FIELD_BWD = [_i32] * 4 + [_ptr] * 7 + [_f32] * 3 + [_ptr] * 10 + [_size, _ptr]
_SDF_NORMAL_BWD = [_i32] * 3 + [_ptr] * 13 + [_size, _ptr]
_DEPTH_MAP = [_i32] * 3 + [_i64] * 2 + [_ptr, _f32, _f32, _ptr]  # N or P, H, W, the depth view, sx, sy, camera
_DEPTH_LOSS_BWD = _DEPTH_MAP + [_ptr] * 2 + [_f32] * 2 + [_ptr] * 5

# every export of include/gsr_b200.h: name -> (restype, argtypes)
SIGNATURES = {
    "gsr_geom_bytes": (_size, [_i32]),
    "gsr_binning_bytes": (_size, [_size]),
    "gsr_image_bytes": (_size, [_i32, _i32]),
    "gsr_binning_capacity": (_size, [_size]),
    "gsr_binning_bytes_slab": (_size, [_size, _i32, _i32, _i32]),
    "gsr_binning_capacity_slab": (_size, [_size, _i32, _i32, _i32]),
    "gsr_forward": (_int, [_frame, _ws] + [_ptr] * 4 + [_int, _ptr]),
    "gsr_forward_multi": (_int, [_frame, _ws] + [_ptr] * 6 + [_int, _ptr]),
    "gsr_axis_normals": (_int, [_i32] + [_ptr] * 4 + [_int, _ptr, _ptr]),
    "gsr_sugar_normals": (_int, [_i32] + [_ptr] * 6),
    "gsr_sugar_normals_backward": (_int, [_i32] + [_ptr] * 7),
    "gsr_sugar_colors": (_int, [_i32] * 3 + [_ptr] * 9),
    "gsr_sugar_colors_backward": (_int, [_i32] * 3 + [_ptr] * 13),
    "gsr_normal_maps": (_int, [_i32, _i32] + [_ptr] * 3 + [_f32] * 4 + [_ptr] * 3),
    "gsr_pack_frame": (_int, [_i32, _i32] + [_ptr] * 4 + [_f32] + [_ptr] * 4),
    "gsr_activate_gaussians": (_int, [_i32, _i32] + [_ptr] * 6 + [C.POINTER(gsr_object_xform)] + [_ptr] * 6),
    "gsr_activate_gaussians_backward": (_int, [_i32, _i32] + [_ptr] * 17),
    "gsr_backward": (_int, [_frame, _ws] + [_ptr] * 5 + [_grads, _ptr]),
    "gsr_backward_multi": (_int, [_frame, _ws] + [_ptr] * 8 + [_grads, _ptr]),
    "gsr_backward_det_bytes": (_size, [_size, _i32, _i32, _int]),
    "gsr_backward_det": (_int, [_frame, _ws] + [_ptr] * 8 + [_grads, _ptr, _size, _ptr]),
    "gsr_mark_visible": (_int, [_i32] + [_ptr] * 5),
    "gsr_dist2_bytes": (_size, [_i32]),
    "gsr_dist2": (_int, [_i32] + [_ptr] * 3 + [_size, _ptr]),
    "gsr_knn_bytes": (_size, [_i32] * 3),
    "gsr_knn": (_int, [_i32] * 3 + [_ptr] * 5 + [_size, _ptr]),
    "gsr_sugar_field_bytes": (_size, [_i32]),
    "gsr_sugar_field": (_int, [_i32] * 4 + [_ptr] * 7 + [_f32] * 3 + [_ptr] * 5 + [_size, _ptr]),
    "gsr_sugar_field_backward": (_int, _FIELD_BWD),
    "gsr_sugar_field_backward_det_bytes": (_size, [_i32] * 3),
    "gsr_sugar_field_backward_det": (_int, _FIELD_BWD),
    "gsr_sugar_sdf_normal_bytes": (_size, [_i32]),
    "gsr_sugar_sdf_normal": (_int, [_i32] * 3 + [_ptr] * 10 + [_size, _ptr]),
    "gsr_sugar_sdf_normal_backward": (_int, _SDF_NORMAL_BWD),
    "gsr_sugar_sdf_normal_backward_det_bytes": (_size, [_i32] * 3 + [_int]),
    "gsr_sugar_sdf_normal_backward_det": (_int, _SDF_NORMAL_BWD),
    "gsr_sugar_sample_bytes": (_size, [_i32]),
    "gsr_sugar_sample": (_int, [_i32, _i32, _f32, _i32] + [_ptr] * 11 + [_size, _ptr]),
    "gsr_sugar_sample_backward": (_int, [_i32, _i32, _f32] + [_ptr] * 10),
    "gsr_sugar_sample_backward_det_bytes": (_size, [_i32] * 2),
    "gsr_sugar_sample_backward_det": (_int, [_i32, _i32, _f32] + [_ptr] * 10 + [_size, _ptr]),
    "gsr_sugar_surface_mask": (_int, _DEPTH_MAP + [_ptr] * 3 + [_f32] + [_ptr] * 3),
    "gsr_sugar_depth_sdf_loss_bytes": (_size, [_i32]),
    "gsr_sugar_depth_sdf_loss": (_int, _DEPTH_MAP + [_ptr] * 2 + [_f32] * 2 + [_ptr] * 3 + [_size, _ptr]),
    "gsr_sugar_depth_sdf_loss_backward": (_int, _DEPTH_LOSS_BWD + [_ptr]),
    "gsr_sugar_depth_sdf_loss_backward_det_bytes": (_size, [_i32] * 3),
    "gsr_sugar_depth_sdf_loss_backward_det": (_int, _DEPTH_LOSS_BWD + [_ptr, _size, _ptr]),
    "gsr_densify_stats": (_int, [_i32] * 2 + [_ptr] * 7),
    "gsr_densify_plan_bytes": (_size, [_i32]),
    "gsr_densify_plan": (_int, [_i32] + [_ptr] * 4 + [_f32] * 3 + [_i32] + [_f32] * 2 + [_ptr] * 3 + [_size, _ptr]),
    "gsr_densify_apply": (_int, [_i32] * 3 + [C.POINTER(gsr_densify_group)] + [_ptr] * 5 + [_i32, _ptr]),
    "gsr_adam_step": (_int, [_i32, C.POINTER(gsr_adam_tensor), _ptr]),
    "gsr_photometric_loss_bytes": (_size, [_i32] * 5),
    "gsr_photometric_loss": (_int, [_i32] * 4 + [_ptr] * 5 + [_i32] + [_ptr] * 3 + [_size, _ptr]),
    "gsr_photometric_loss_backward": (_int, [_i32] * 4 + [_ptr] * 9 + [_size, _ptr]),
    "gsr_normal_loss": (_int, [_i64] + [_ptr] * 5 + [_i64, _f32, _ptr, _ptr, _size, _ptr]),
    "gsr_normal_loss_backward": (_int, [_i64] + [_ptr] * 5 + [_i64, _f32] + [_ptr] * 3 + [_size, _ptr]),
    "gsr_anisotropic_loss": (_int, [_i64, _ptr, _f32, _ptr, _ptr, _size, _ptr]),
    "gsr_anisotropic_loss_backward": (_int, [_i64, _ptr, _f32] + [_ptr] * 3),
    "gsr_depth_loss": (_int, [_i64, _ptr, _i64, _ptr, _i64, _f32, _ptr, _ptr, _size, _ptr]),
    "gsr_depth_loss_backward": (_int, [_i64, _ptr, _i64, _ptr, _i64, _f32] + [_ptr] * 3 + [_size, _ptr]),
    "gsr_opacity_loss": (_int, [_i64, _ptr, _i64, _ptr, _ptr, _size, _ptr]),
    "gsr_opacity_loss_backward": (_int, [_i64] + [_ptr] * 3),
    "gsr_sparsity_loss": (_int, [_i64, _ptr, _i64, _ptr, _ptr, _size, _ptr]),
    "gsr_sparsity_loss_backward": (_int, [_i64, _ptr, _i64] + [_ptr] * 3),
    "gsr_entropy_loss": (_int, [_i64, _ptr, _i64, _ptr, _i64, _ptr, _ptr, _size, _ptr]),
    "gsr_entropy_loss_backward": (_int, [_i64, _ptr, _i64, _ptr, _i64] + [_ptr] * 3 + [_size, _ptr]),
    "gsr_density_estimation_loss": (_int, [_i64, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32, _ptr, _ptr, _size, _ptr]),
    "gsr_density_estimation_loss_backward": (_int, [_i64, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32] + [_ptr] * 5),
    "gsr_percentile_low": (_int, [_i64] + [_ptr] * 3 + [_size, _ptr]),
    "gsr_composite": (_int, [_i32] * 2 + [_ptr] * 14),
    "gsr_select_rows_bytes": (_size, [_i64]),
    "gsr_select_rows": (_int, [_i64] + [_ptr] * 11 + [_size, _ptr]),
    "gsr_pack_masks": (_int, [_i32] * 3 + [_ptr] * 3),
    "gsr_mask_disagreement": (_int, [_i32] * 2 + [_ptr] * 2 + [_f32, _ptr, _ptr]),
    "gsr_png_bound": (_size, [_i32] * 3),
    "gsr_png_workspace_bytes": (_size, [_i32, C.POINTER(gsr_png_image)]),
    "gsr_png_encode": (_int, [C.POINTER(gsr_png_image), _i32, C.POINTER(C.c_void_p), _ptr, _ptr, _size, _ptr]),
    "gsr_mesh_bvh_bytes": (_size, [_i32]),
    "gsr_mesh_build_bytes": (_size, [_i32]),
    "gsr_mesh_build": (_int, [_i64, _i32] + [_ptr] * 3 + [_size, _ptr, _size, _ptr]),
    "gsr_mesh_first_hit": (_int, [_i32, _ptr, _i64, _ptr, _ptr, _i32] + [_ptr] * 4),
    "gsr_mesh_inpaint_mask": (_int, [_i64, _ptr, _ptr, _i32] + [_ptr] * 8),
    "gsr_mesh_closest_bytes": (_size, [_i64]),
    "gsr_mesh_closest": (_int, [_i32, _ptr, _i64, _ptr, _i32, _ptr, _ptr, _ptr, _size, _ptr]),
    "gsr_mesh_isin_rows_bytes": (_size, [_i64, _i32]),
    "gsr_mesh_isin_rows": (_int, [_i64, _ptr, _i64, _ptr, _i32, _i32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(_i32), _ptr,
                                  _ptr, _size, _ptr]),
    "gsr_get_views": (_int, [_ws, _i32, _i32, _i32, C.POINTER(gsr_views)]),
    "gsr_profile_begin": (_int, [_int]),
    "gsr_profile_begin_strided": (_int, [_int, _int]),
    "gsr_profile_end": (_int, [C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "gsr_last_error": (C.c_char_p, []),
    "gsr_abi_version": (_int, []),
}
EXPORTS = tuple(SIGNATURES)


def _load() -> C.CDLL:
    path = _build.SO_PATH
    if _build.is_stale():
        # rebuild where a toolkit exists; a stale prebuilt library is still used on a box without nvcc
        try:
            _build.build()
        except Exception as ex:  # noqa: BLE001
            if not os.path.exists(path):
                raise ImportError("autovfx_b200: CUDA library %s is missing and cannot be built (%s). "
                                  "There is no CPU fallback." % (path, ex)) from ex
    lib = C.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        if not hasattr(lib, name):
            raise ImportError("autovfx_b200: %s does not export %s" % (path, name))
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.gsr_abi_version() != ABI_VERSION:
        raise ImportError("autovfx_b200: ABI mismatch, rebuild with `python -m autovfx_b200.build --force`")
    return lib


lib = _load()


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib.gsr_last_error().decode("utf-8", "replace")))


def scratch_bytes(nbytes: int, device: torch.device) -> torch.Tensor:
    """A byte buffer from the caching allocator, without the NaN fill torch gives every torch.empty under
    use_deterministic_algorithms: the library's deterministic backwards (gsr_backward_det, gsr_sugar_*_backward_det) write every
    scratch byte they read, and a fill of gigabytes would cost about as much as the backward itself."""
    fill = torch.utils.deterministic.fill_uninitialized_memory
    torch.utils.deterministic.fill_uninitialized_memory = False
    try:
        return torch.empty(nbytes, dtype=torch.uint8, device=device)
    finally:
        torch.utils.deterministic.fill_uninitialized_memory = fill


def stream_ptr(device) -> C.c_void_p:
    """PyTorch's current stream on ``device``, as the ``cudaStream_t`` argument of a library call."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
