"""ctypes binding of libfrosting_b200.so (the C ABI in include/frosting_b200.h).

There is no fallback: if the CUDA library is missing this module raises at import of the symbols,
and every op in this package fails loudly.  PyTorch is used only for device memory and streams.
"""
import ctypes as C
import math
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfrosting_b200.so")

FB200_STATUS_WORDS = 8
ST_NUM_RENDERED, ST_OVERFLOW, ST_MAX_TILE, ST_NUM_VISIBLE = 0, 1, 2, 3
TILE = 16
NUM_STAGES = 5
ABI_VERSION = 9
STAGES = ("preprocess", "binning", "render_fwd", "render_bwd", "geom_bwd")


class Params(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("sh_degree", C.c_int32), ("sh_coeffs", C.c_int32),
        ("image_width", C.c_int32), ("image_height", C.c_int32),
        ("tanfovx", C.c_float), ("tanfovy", C.c_float), ("scale_modifier", C.c_float),
        ("prefiltered", C.c_int32), ("debug", C.c_int32),
        ("extra", C.c_void_p),          # const fb200_extra* (row f4) or NULL
    ]


class Extra(C.Structure):
    _fields_ = [("channels", C.c_int32), ("d_features", C.c_void_p), ("d_background", C.c_void_p),
                ("d_out", C.c_void_p), ("d_dL_dout", C.c_void_p), ("d_dL_dfeatures", C.c_void_p)]


class Inputs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "d_background", "d_means3D", "d_shs", "d_colors_precomp", "d_opacities", "d_scales",
        "d_rotations", "d_cov3D_precomp", "d_viewmatrix", "d_projmatrix", "d_campos", "d_visibility",
        "d_point_cells", "d_face_visible")] + [("n_cell_points", C.c_int64),
                                               ("frosting", C.c_void_p)]     # const fb200_frosting_params* or NULL


class Workspace(C.Structure):
    _fields_ = [
        ("d_geom", C.c_void_p), ("geom_bytes", C.c_size_t),
        ("d_image", C.c_void_p), ("image_bytes", C.c_size_t),
        ("d_binning", C.c_void_p), ("binning_bytes", C.c_size_t),
        ("binning_capacity", C.c_int64),
        ("d_status", C.c_void_p),
        ("acc_zeroed_by_forward", C.c_int32),
        ("h_status", C.c_void_p),
    ]


class Grads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "d_dL_dmeans2D", "d_dL_dcolors", "d_dL_dopacity", "d_dL_dmeans3D", "d_dL_dcov3D", "d_dL_dsh",
        "d_dL_dscales", "d_dL_drotations")] + [("sparse_rows", C.c_int32),
                                               ("frosting", C.c_void_p)]   # const fb200_frosting_grads* or NULL


class FrostingParams(C.Structure):
    _fields_ = [("P", C.c_int32), ("n_verts", C.c_int32), ("n_faces", C.c_int32), ("sh_rest", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("d_bary_logits", "d_cells", "d_faces", "d_inner_verts", "d_outer_verts",
                                          "d_opacity_logits", "d_log_scales", "d_quats", "d_sh_dc", "d_sh_rest",
                                          "d_mask", "d_face_visible", "d_radii")] + \
               [("n_bg", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("d_bg_points", "d_bg_opacity_logits", "d_bg_log_scales", "d_bg_quats",
                                          "d_bg_sh_dc", "d_bg_sh_rest")]


class FrostingGrads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("d_bary_logits", "d_inner_verts", "d_outer_verts", "d_opacity_logits",
                                          "d_log_scales", "d_quats", "d_sh_dc", "d_sh_rest", "d_bg_points",
                                          "d_bg_opacity_logits", "d_bg_log_scales", "d_bg_quats", "d_bg_sh_dc",
                                          "d_bg_sh_rest")]


RESCALE_MEDIAN, RESCALE_TRIANGLE = 0, 1
EDIT_SELECT_WORDS = 2051


class FrostingEdit(C.Structure):
    _fields_ = [("n_verts", C.c_int32), ("n_faces", C.c_int32), ("rescaling", C.c_int32), ("n_edited", C.c_int32),
                ("deformation_threshold", C.c_float)] + \
               [(n, C.c_void_p) for n in ("d_base_verts", "d_faces", "d_inner_dist", "d_outer_dist", "d_edition_mask",
                                          "d_verts_edition_mask", "d_vf_offsets", "d_vf_faces", "d_ref_quats",
                                          "d_ref_dists", "d_ref_median", "d_dists", "d_face_normals", "d_rel_quats",
                                          "d_face_factor", "d_face_keep", "d_factor", "d_select", "d_inner_verts",
                                          "d_outer_verts")]


class FrostingSkin(C.Structure):
    _fields_ = [("n_rows", C.c_int32), ("n_verts", C.c_int32), ("n_bones", C.c_int32), ("n_frames", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("d_tpose", "d_vert_ids", "d_offsets", "d_bones", "d_weights", "d_reset",
                                          "d_pose")]


class Texture(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_faces", "n_points", "square_size", "n_square_per_axis", "texture_size")] + \
               [(n, C.c_void_p) for n in ("d_cell_offsets", "d_cell_points", "d_sh_dc", "d_face_sh", "d_face_acc",
                                          "d_texel_acc", "d_face_winner", "d_texel_winner")]


class SugarReg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("P", "K", "N")] + [("sampling_scale_factor", C.c_float)] + \
               [(n, C.c_void_p) for n in ("d_points", "d_scaling", "d_quaternions", "d_strengths", "d_knn_idx", "d_idx",
                                          "d_eps", "d_workspace")]


class FrostingInit(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_verts", "n_faces", "P", "K", "n_samples", "smooth_K", "std_K")] + \
               [(n, C.c_float) for n in ("level", "std_range", "min_layer", "half_layer")] + \
               [(n, C.c_void_p) for n in ("d_verts", "d_faces", "d_vf_offsets", "d_vf_faces", "d_normals", "d_points",
                                          "d_scaling", "d_quaternions", "d_strengths", "d_knn_idx", "d_std_idx",
                                          "d_inner_range", "d_outer_range", "d_min_clamp_inner", "d_max_clamp_outer",
                                          "d_fractions", "d_smooth_idx", "d_level_outer", "d_level_inner",
                                          "d_outer_dist", "d_inner_dist", "d_outer_verts", "d_inner_verts",
                                          "d_densities")]


TRIM_K = 8


class FrostingCreate(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_verts", "n_faces", "n_iterations", "n_gaussians", "n_gs", "sh_rest",
                                         "contract")] + \
               [(n, C.c_float) for n in ("step", "inside_th", "extent", "min_height")] + \
               [(n, C.c_void_p) for n in ("d_verts", "d_faces", "d_normals", "d_inner_init", "d_outer_init",
                                          "d_inner_verts", "d_outer_verts", "d_inner_dist", "d_outer_dist",
                                          "d_inner_stop", "d_outer_stop", "d_shell", "d_centres", "d_knn_workspace")] + \
               [("knn_workspace_bytes", C.c_size_t)] + \
               [(n, C.c_void_p) for n in ("d_knn_dists", "d_knn_idx", "d_camera_center", "d_volumes", "d_cells", "d_u",
                                          "d_bary_logits", "d_points", "d_max_scales", "d_nn_idx", "d_sh_idx",
                                          "d_gs_sh_dc", "d_gs_sh_rest", "d_dist2", "d_log_scales", "d_quats",
                                          "d_opacity_logits", "d_sh_dc", "d_sh_rest")]


ADAM_MAX_GROUPS = 16
MAX_PEERS = 8
PEER_HANDLE_BYTES = 64


class AdamArgs(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32),
                ("peer_params", C.c_void_p * MAX_PEERS), ("peer_grads", C.c_void_p * MAX_PEERS),
                ("d_exp_avg", C.c_void_p), ("d_exp_avg_sq", C.c_void_p),
                ("shard_lo", C.c_int64), ("shard_hi", C.c_int64), ("n_groups", C.c_int32),
                ("group_start", C.c_int64 * (ADAM_MAX_GROUPS + 1)), ("lr", C.c_float * ADAM_MAX_GROUPS),
                ("beta1", C.c_double), ("beta2", C.c_double), ("eps", C.c_float),
                ("bias_correction1", C.c_float), ("bias_correction2_sqrt", C.c_float), ("grad_scale", C.c_float),
                ("mc_grads", C.c_void_p), ("mc_params", C.c_void_p),
                ("peer_row_radii", C.c_void_p * MAX_PEERS), ("row_width", C.c_int32 * ADAM_MAX_GROUPS),
                ("row_count", C.c_int32)]


class Layout(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in (
        "geom_rec", "geom_depth", "geom_rect", "geom_clamped", "img_final_T", "img_n_contrib",
        "img_ranges", "img_tile_count", "bin_point_list", "bin_keys", "geom_acc", "img_last_entry", "bin_sub_hits")]


def workspace_views(geom, image, binning, P, W, H, capacity, R):
    """Named tensor views of a frame's workspace sub-arrays, as the library carved them: `fb200_get_layout` offsets from
    each buffer's first 128-byte aligned byte.  The layout follows from `capacity`; the binning views are R entries
    long.  A buffer given as None contributes no views."""
    lay = Layout()
    check(lib().fb200_get_layout(P, W, H, capacity, C.byref(lay)))
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    table = (  # name, buffer, fb200_layout field, dtype, shape
        ("rec", geom, "geom_rec", torch.float32, (P, 12)),
        ("depth", geom, "geom_depth", torch.float32, (P,)),
        ("rect", geom, "geom_rect", torch.int32, (P, 2)),
        ("clamped", geom, "geom_clamped", torch.uint8, (P,)),
        ("acc", geom, "geom_acc", torch.float32, (P, 12)),
        ("final_T", image, "img_final_T", torch.float32, (H, W)),
        ("n_contrib", image, "img_n_contrib", torch.int32, (H, W)),
        ("last_entry", image, "img_last_entry", torch.int32, (H, W)),
        ("ranges", image, "img_ranges", torch.int32, (T, 2)),
        ("tile_count", image, "img_tile_count", torch.int32, (T,)),
        ("point_list", binning, "bin_point_list", torch.int32, (R,)),
        ("keys", binning, "bin_keys", torch.int64, (R,)),
        ("sub_hits", binning, "bin_sub_hits", torch.int32, (8 * R,)),   # 8 sub-tile hit lists per tile
    )
    views = {}
    for name, buf, field, dtype, shape in table:
        if buf is None:
            continue
        start = (-buf.data_ptr()) % 128 + getattr(lay, field)
        views[name] = buf[start:start + math.prod(shape) * dtype.itemsize].view(dtype).view(shape)
    return views


# (C struct, ctypes mirror) in the order fb200_abi_struct_sizes reports them (FB200_ABI_STRUCTS)
ABI_STRUCTS = (
    ("fb200_params", Params), ("fb200_inputs", Inputs), ("fb200_workspace", Workspace), ("fb200_grads", Grads),
    ("fb200_extra", Extra), ("fb200_frosting_params", FrostingParams), ("fb200_frosting_grads", FrostingGrads),
    ("fb200_adam_args", AdamArgs), ("fb200_layout", Layout), ("fb200_frosting_edit", FrostingEdit),
    ("fb200_frosting_skin", FrostingSkin), ("fb200_texture", Texture), ("fb200_sugar_reg", SugarReg),
    ("fb200_frosting_init", FrostingInit), ("fb200_frosting_create", FrostingCreate),
)

_i32, _i64, _f32, _vp, _int, _size = C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_int, C.c_size_t
_frame = [C.POINTER(Params), C.POINTER(Inputs), C.POINTER(Workspace)]

# name -> (restype, argtypes) of every function include/frosting_b200.h declares; tests/test_abi_cpu.py checks each
# against its prototype
SIGNATURES = {
    "fb200_geom_bytes": (_size, [_i32]),
    "fb200_image_bytes": (_size, [_i32, _i32]),
    "fb200_binning_bytes": (_size, [_i64]),
    "fb200_forward": (_int, _frame + [_vp, _vp, _vp]),
    "fb200_forward_geometry": (_int, _frame + [_vp, _vp]),
    "fb200_forward_raster": (_int, _frame + [_vp, _vp, _vp]),
    "fb200_backward": (_int, _frame + [_vp, _vp, C.POINTER(Grads), _vp]),
    "fb200_mark_visible": (_int, [_i32, _vp, _vp, _vp, _vp, _vp]),
    "fb200_mesh_visibility": (_int, [_i32, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i32, _vp, _vp]),
    "fb200_gaussian_mask_from_faces": (_int, [_i32, _vp, _i32, _vp, _i32, _vp, _vp]),
    "fb200_frosting_attributes": (_int, [C.POINTER(FrostingParams)] + [_vp] * 6),
    "fb200_frosting_attributes_backward": (_int, [C.POINTER(FrostingParams)] + [_vp] * 5 +
                                           [C.POINTER(FrostingGrads), _vp]),
    "fb200_frosting_edit_shell": (_int, [C.POINTER(FrostingEdit), _vp]),
    "fb200_frosting_edit_attributes": (_int, [C.POINTER(FrostingEdit), C.POINTER(FrostingParams), _i32] + [_vp] * 8),
    "fb200_frosting_edit_complex_capture": (_int, [C.POINTER(FrostingEdit), C.POINTER(FrostingParams)] + [_vp] * 4),
    "fb200_frosting_edit_attributes_complex": (_int, [C.POINTER(FrostingEdit), C.POINTER(FrostingParams), _i32] +
                                               [_vp] * 10),
    "fb200_frosting_skin_pose": (_int, [C.POINTER(FrostingSkin), _i32, _vp, _vp]),
    "fb200_mesh_barycentrics": (_int, [_i32, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "fb200_texture_face_sh_colours": (_int, [C.POINTER(Texture), _vp]),
    "fb200_texture_add_view": (_int, [C.POINTER(Texture), _vp, _vp, _vp, _i32, _i32, _vp]),
    "fb200_texture_finish": (_int, [C.POINTER(Texture), _vp, _vp]),
    "fb200_loss_partials": (_size, [_i32, _i32, _i32]),
    "fb200_l1_dssim_forward": (_int, [_vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp]),
    "fb200_l1_dssim_backward": (_int, [_vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp]),
    "fb200_sugar_reg_workspace_bytes": (_size, [_i32, _i32, _i32, _i32]),
    "fb200_sugar_reg_forward": (_int, [C.POINTER(SugarReg), _i32, _vp, _vp]),
    "fb200_sugar_reg_backward": (_int, [C.POINTER(SugarReg)] + [_vp] * 6),
    "fb200_sugar_dn_features": (_int, [_i32] + [_vp] * 7),
    "fb200_sugar_dn_features_backward": (_int, [_i32] + [_vp] * 9),
    "fb200_sugar_dn_partials": (_size, [_i32, _i32]),
    "fb200_sugar_dn_loss_forward": (_int, [_vp, _i32, _i32] + [_vp] * 5),
    "fb200_sugar_dn_loss_backward": (_int, [_vp, _i32, _i32] + [_vp] * 5),
    "fb200_knn_workspace_bytes": (_size, [_i32, _i32, _i32]),
    "fb200_knn": (_int, [_vp, _i32, _vp, _i32, _i32, _vp, _size, _vp, _vp, _vp]),
    "fb200_level_points": (_int, [C.POINTER(FrostingInit), _vp]),
    "fb200_frosting_trim": (_int, [C.POINTER(FrostingCreate), _vp]),
    "fb200_frosting_volumes": (_int, [C.POINTER(FrostingCreate), _vp]),
    "fb200_frosting_sample": (_int, [C.POINTER(FrostingCreate), _vp]),
    "fb200_frosting_finish": (_int, [C.POINTER(FrostingCreate), _vp]),
    "fb200_adam_step": (_int, [C.POINTER(AdamArgs), _vp]),
    "fb200_peer_alloc": (_int, [_size, C.POINTER(_vp)]),
    "fb200_peer_free": (_int, [_vp]),
    "fb200_peer_export": (_int, [_vp, C.c_char_p]),
    "fb200_peer_open": (_int, [C.c_char_p, C.POINTER(_vp)]),
    "fb200_peer_close": (_int, [_vp]),
    "fb200_get_layout": (_int, [_i32, _i32, _i32, _i64, C.POINTER(Layout)]),
    "fb200_profile_enable": (_int, [_i32]),
    "fb200_profile_read": (_int, [C.POINTER(_f32)]),
    "fb200_kernel_launches": (_i64, []),
    "fb200_last_error": (C.c_char_p, []),
    "fb200_abi_version": (_int, []),
    "fb200_abi_struct_sizes": (_int, [C.POINTER(_size)]),
}
EXPORTED = list(SIGNATURES)

_lib = None


def build_if_needed():
    """(Re)build the shared library in-tree when sources are newer; needs nvcc only."""
    from . import build as _build
    return _build.build()


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        try:
            build_if_needed()
        except Exception as ex:  # no nvcc / compile error: fail loudly, never fall back
            raise RuntimeError(
                f"frosting_b200: CUDA library {LIB_PATH} is missing and could not be built ({ex}). "
                "Run `python -m frosting_b200.build`. There is no CPU fallback.") from ex
    L = C.CDLL(LIB_PATH)
    # before anything else: the exported names and the struct count depend on the version (an int(void) function,
    # callable with ctypes' default signature)
    if L.fb200_abi_version() != ABI_VERSION:
        raise RuntimeError("frosting_b200: ABI version mismatch between header and library")
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    sizes = (C.c_size_t * len(ABI_STRUCTS))()
    if L.fb200_abi_struct_sizes(sizes) != 0 or list(sizes) != [C.sizeof(m) for _, m in ABI_STRUCTS]:
        raise RuntimeError("frosting_b200: ctypes struct mirrors out of sync with include/frosting_b200.h: " +
                           ", ".join(f"{n} {s} vs {C.sizeof(m)}" for (n, m), s in zip(ABI_STRUCTS, sizes)))
    _lib = L
    return L


def profile_enable(on: bool):
    check(lib().fb200_profile_enable(1 if on else 0))


def profile_read():
    """Device milliseconds per stage of the most recent forward/backward on this thread."""
    buf = (C.c_float * NUM_STAGES)()
    check(lib().fb200_profile_read(buf))
    return {n: float(buf[i]) for i, n in enumerate(STAGES)}


def kernel_launches() -> int:
    return int(lib().fb200_kernel_launches())


def ptr(t):
    """A tensor's device pointer as a `d_*` argument: NULL for a missing or empty tensor."""
    return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())


def stream(device):
    """The current CUDA stream of `device` as the `void* stream` argument."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Fb200Error(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        msg = lib().fb200_last_error().decode("utf-8", "replace")
        raise Fb200Error(f"frosting_b200 error {rc}: {msg}")
