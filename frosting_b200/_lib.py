"""ctypes binding of libfrosting_b200.so (the C ABI in include/frosting_b200.h).

There is no fallback: if the CUDA library is missing this module raises at import of the symbols,
and every op in this package fails loudly.  PyTorch is used only for device memory and streams.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfrosting_b200.so")

FB200_STATUS_WORDS = 8
ST_NUM_RENDERED, ST_OVERFLOW, ST_MAX_TILE, ST_NUM_VISIBLE = 0, 1, 2, 3
TILE = 16

# every symbol include/frosting_b200.h declares
EXPORTED = [
    "fb200_abi_version", "fb200_abi_struct_sizes", "fb200_last_error", "fb200_geom_bytes", "fb200_image_bytes",
    "fb200_binning_bytes", "fb200_forward", "fb200_forward_geometry", "fb200_forward_raster", "fb200_backward", "fb200_mark_visible",
    "fb200_mesh_visibility", "fb200_gaussian_mask_from_faces", "fb200_get_layout",
    "fb200_profile_enable", "fb200_profile_read", "fb200_kernel_launches",
    "fb200_frosting_attributes", "fb200_frosting_attributes_backward",
    "fb200_frosting_edit_shell", "fb200_frosting_edit_attributes", "fb200_frosting_edit_struct_size",
    "fb200_frosting_edit_complex_capture", "fb200_frosting_edit_attributes_complex",
    "fb200_frosting_skin_pose", "fb200_frosting_skin_struct_size",
    "fb200_mesh_barycentrics", "fb200_texture_face_sh_colours", "fb200_texture_add_view", "fb200_texture_finish",
    "fb200_texture_struct_size",
    "fb200_loss_partials", "fb200_l1_dssim_forward", "fb200_l1_dssim_backward",
    "fb200_sugar_reg_workspace_bytes", "fb200_sugar_reg_forward", "fb200_sugar_reg_backward",
    "fb200_sugar_reg_struct_size",
    "fb200_adam_step", "fb200_peer_alloc", "fb200_peer_free", "fb200_peer_export", "fb200_peer_open", "fb200_peer_close",
]
NUM_STAGES = 5
ABI_VERSION = 7
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
        "img_ranges", "img_tile_count", "bin_point_list", "bin_keys", "geom_acc")]


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
    L.fb200_abi_version.restype = C.c_int
    L.fb200_last_error.restype = C.c_char_p
    for n in ("fb200_geom_bytes", "fb200_image_bytes", "fb200_binning_bytes"):
        getattr(L, n).restype = C.c_size_t
    L.fb200_geom_bytes.argtypes = [C.c_int32]
    L.fb200_image_bytes.argtypes = [C.c_int32, C.c_int32]
    L.fb200_binning_bytes.argtypes = [C.c_int64]
    L.fb200_forward.argtypes = [C.POINTER(Params), C.POINTER(Inputs), C.POINTER(Workspace),
                                C.c_void_p, C.c_void_p, C.c_void_p]
    L.fb200_forward_geometry.argtypes = [C.POINTER(Params), C.POINTER(Inputs), C.POINTER(Workspace),
                                         C.c_void_p, C.c_void_p]
    L.fb200_forward_raster.argtypes = [C.POINTER(Params), C.POINTER(Inputs), C.POINTER(Workspace),
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    L.fb200_backward.argtypes = [C.POINTER(Params), C.POINTER(Inputs), C.POINTER(Workspace),
                                 C.c_void_p, C.c_void_p, C.POINTER(Grads), C.c_void_p]
    L.fb200_mark_visible.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fb200_mesh_visibility.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int32, C.c_void_p, C.c_void_p]
    L.fb200_gaussian_mask_from_faces.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                                 C.c_void_p, C.c_void_p]
    L.fb200_get_layout.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.POINTER(Layout)]
    L.fb200_frosting_attributes.argtypes = [C.POINTER(FrostingParams)] + [C.c_void_p] * 6
    L.fb200_frosting_attributes.restype = C.c_int
    L.fb200_frosting_attributes_backward.argtypes = [C.POINTER(FrostingParams)] + [C.c_void_p] * 5 + \
        [C.POINTER(FrostingGrads), C.c_void_p]
    L.fb200_frosting_attributes_backward.restype = C.c_int
    L.fb200_frosting_edit_shell.argtypes = [C.POINTER(FrostingEdit), C.c_void_p]
    L.fb200_frosting_edit_shell.restype = C.c_int
    L.fb200_frosting_edit_attributes.argtypes = [C.POINTER(FrostingEdit), C.POINTER(FrostingParams), C.c_int32] + \
        [C.c_void_p] * 8
    L.fb200_frosting_edit_attributes.restype = C.c_int
    L.fb200_frosting_edit_struct_size.restype = C.c_size_t
    L.fb200_frosting_edit_complex_capture.argtypes = [C.POINTER(FrostingEdit), C.POINTER(FrostingParams)] + \
        [C.c_void_p] * 4
    L.fb200_frosting_edit_complex_capture.restype = C.c_int
    L.fb200_frosting_edit_attributes_complex.argtypes = [C.POINTER(FrostingEdit), C.POINTER(FrostingParams),
                                                         C.c_int32] + [C.c_void_p] * 10
    L.fb200_frosting_edit_attributes_complex.restype = C.c_int
    L.fb200_frosting_skin_pose.argtypes = [C.POINTER(FrostingSkin), C.c_int32, C.c_void_p, C.c_void_p]
    L.fb200_frosting_skin_pose.restype = C.c_int
    L.fb200_frosting_skin_struct_size.restype = C.c_size_t
    L.fb200_mesh_barycentrics.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                          C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fb200_texture_face_sh_colours.argtypes = [C.POINTER(Texture), C.c_void_p]
    L.fb200_texture_add_view.argtypes = [C.POINTER(Texture), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_void_p]
    L.fb200_texture_finish.argtypes = [C.POINTER(Texture), C.c_void_p, C.c_void_p]
    for n in ("fb200_mesh_barycentrics", "fb200_texture_face_sh_colours", "fb200_texture_add_view",
              "fb200_texture_finish"):
        getattr(L, n).restype = C.c_int
    L.fb200_texture_struct_size.restype = C.c_size_t
    L.fb200_loss_partials.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    L.fb200_loss_partials.restype = C.c_size_t
    L.fb200_l1_dssim_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fb200_l1_dssim_forward.restype = C.c_int
    L.fb200_l1_dssim_backward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fb200_l1_dssim_backward.restype = C.c_int
    L.fb200_sugar_reg_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    L.fb200_sugar_reg_workspace_bytes.restype = C.c_size_t
    L.fb200_sugar_reg_forward.argtypes = [C.POINTER(SugarReg), C.c_int32, C.c_void_p, C.c_void_p]
    L.fb200_sugar_reg_forward.restype = C.c_int
    L.fb200_sugar_reg_backward.argtypes = [C.POINTER(SugarReg)] + [C.c_void_p] * 6
    L.fb200_sugar_reg_backward.restype = C.c_int
    L.fb200_sugar_reg_struct_size.restype = C.c_size_t
    L.fb200_adam_step.argtypes = [C.POINTER(AdamArgs), C.c_void_p]
    L.fb200_peer_alloc.argtypes = [C.c_size_t, C.POINTER(C.c_void_p)]
    L.fb200_peer_free.argtypes = [C.c_void_p]
    L.fb200_peer_export.argtypes = [C.c_void_p, C.c_char_p]
    L.fb200_peer_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
    L.fb200_peer_close.argtypes = [C.c_void_p]
    for n in ("fb200_adam_step", "fb200_peer_alloc", "fb200_peer_free", "fb200_peer_export", "fb200_peer_open",
              "fb200_peer_close"):
        getattr(L, n).restype = C.c_int
    L.fb200_profile_enable.argtypes = [C.c_int32]
    L.fb200_profile_enable.restype = C.c_int
    L.fb200_profile_read.argtypes = [C.POINTER(C.c_float)]
    L.fb200_profile_read.restype = C.c_int
    L.fb200_kernel_launches.restype = C.c_int64
    for n in ("fb200_forward", "fb200_forward_geometry", "fb200_forward_raster", "fb200_backward", "fb200_mark_visible", "fb200_mesh_visibility",
              "fb200_gaussian_mask_from_faces", "fb200_get_layout"):
        getattr(L, n).restype = C.c_int
    if L.fb200_abi_version() != ABI_VERSION:
        raise RuntimeError("frosting_b200: ABI version mismatch between header and library")
    mirrors = (Params, Inputs, Workspace, Grads, Extra, FrostingParams, FrostingGrads, AdamArgs, Layout)
    sizes = (C.c_size_t * len(mirrors))()
    L.fb200_abi_struct_sizes.argtypes = [C.POINTER(C.c_size_t)]
    L.fb200_abi_struct_sizes.restype = C.c_int
    if L.fb200_abi_struct_sizes(sizes) != 0 or [int(x) for x in sizes] != [C.sizeof(m) for m in mirrors]:
        raise RuntimeError("frosting_b200: ctypes struct mirrors out of sync with include/frosting_b200.h: "
                           f"{[int(x) for x in sizes]} vs {[C.sizeof(m) for m in mirrors]}")
    if L.fb200_frosting_edit_struct_size() != C.sizeof(FrostingEdit):
        raise RuntimeError("frosting_b200: ctypes mirror of fb200_frosting_edit out of sync with include/frosting_b200.h")
    if L.fb200_frosting_skin_struct_size() != C.sizeof(FrostingSkin):
        raise RuntimeError("frosting_b200: ctypes mirror of fb200_frosting_skin out of sync with include/frosting_b200.h")
    if L.fb200_texture_struct_size() != C.sizeof(Texture):
        raise RuntimeError("frosting_b200: ctypes mirror of fb200_texture out of sync with include/frosting_b200.h")
    if L.fb200_sugar_reg_struct_size() != C.sizeof(SugarReg):
        raise RuntimeError("frosting_b200: ctypes mirror of fb200_sugar_reg out of sync with include/frosting_b200.h")
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
