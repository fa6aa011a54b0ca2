"""frosting_b200 -- differentiable Gaussian-splatting rasterizer in hand-written CUDA for the H100 (sm_90a).

A drop-in for the render path of Anttwo/Frosting: the `diff_gaussian_rasterization` Python surface
(GaussianRasterizationSettings / GaussianRasterizer) and the mesh occlusion-culling prepass, backed
by hand-written CUDA behind the C ABI of include/frosting_b200.h.  See DESIGN.md / INTEGRATION.md.
"""
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians,
                         forward_with_state)
from .frosting_render import frosting_attributes_fused, frosting_render, frosting_render_two_step
from .edit import FrostingEdit, FrostingEditComplex, frosting_render_edited
from .skin import FrostingSkin, skin_tables
from .texture import TextureBaker, compute_textured_mesh, mesh_bary, write_textured_obj
from .loss import l1_dssim_loss
from .sugar import SugarNeighbours, sample_in_gaussians, sdf_regularization
from .sugar_dn import depth_normal_consistency, depth_normal_features
from .knn import KNN, knn_points
from .frosting_init import LevelPoints, initial_shell, level_points_along_normals
from .frosting_create import GS_KEYS, Trimmed, create_frosting, trim_shell
from .optim import FrostingAdam, OptimizationParams
from .mesh import (MeshRasterizer, RasterizationSettings, Fragments, nvdiff_rasterization,
                   nvdiff_rasterization_with_pix_to_face, rasterize_mesh, gaussian_render_mask)

__all__ = [
    "GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "forward_with_state",
    "MeshRasterizer", "RasterizationSettings", "Fragments", "nvdiff_rasterization",
    "nvdiff_rasterization_with_pix_to_face", "rasterize_mesh", "gaussian_render_mask",
    "install_as_diff_gaussian_rasterization", "frosting_attributes_fused", "frosting_render", "frosting_render_two_step", "FrostingEdit", "FrostingEditComplex", "frosting_render_edited", "FrostingSkin", "skin_tables", "TextureBaker", "compute_textured_mesh", "mesh_bary", "write_textured_obj", "l1_dssim_loss", "SugarNeighbours", "sample_in_gaussians", "sdf_regularization", "depth_normal_features", "depth_normal_consistency", "KNN", "knn_points", "LevelPoints", "initial_shell", "level_points_along_normals", "GS_KEYS", "Trimmed", "create_frosting", "trim_shell", "FrostingAdam", "OptimizationParams",
]


def install_as_diff_gaussian_rasterization():
    """Make `import diff_gaussian_rasterization` resolve to this package (no edit of the caller's tree).

    Equivalent to putting frosting_b200/compat on sys.path; the reference's own backend switch is a
    source-level bool (frosting_scene/frosting_model.py:23), this is the import-site equivalent."""
    import sys
    from .compat import diff_gaussian_rasterization as shim
    sys.modules["diff_gaussian_rasterization"] = shim
    return shim
