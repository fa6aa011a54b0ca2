"""The thickness of a new Frosting layer -- host side of csrc/frosting_init.cu.

`Frosting.__init__` (frosting_scene/frosting_model.py:296-369) decides how thick the frosting is at every base-mesh vertex:
it looks for the level crossings of the coarse SuGaR model's density along each vertex normal inside +-3 sigma, widens
that proposal threefold and looks again in the 3DGS model's density, clamped to a tenth of the proposal.  Here, without
pytorch3d:

    outer_dist, inner_dist, outer_verts, inner_verts = initial_shell(
        (sugar.points, sugar.scaling, sugar.quaternions, sugar.strengths),
        (gs.get_xyz, gs.get_scaling, gs.get_rotation, gs.get_opacity), verts, faces, spatial_extent)

Each pass is one `fb200_level_points` call (two kernels) after its `knn_points` tables.  `torch_reference` restates the
reference's chunked torch computation for any dtype: the float32 comparison route of the tests and the benchmark.
"""
import ctypes as C
from collections import namedtuple

import torch

from . import _lib
from ._lib import ptr, stream
from .knn import knn_points

LevelPoints = namedtuple("LevelPoints", "outer_dist inner_dist outer_verts inner_verts")
MAX_SAMPLES = 32


def _rows(t, name, dev, width):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise ValueError(f"{name} must be a float32 tensor, got "
                         f"{t.dtype if isinstance(t, torch.Tensor) else type(t).__name__}")
    if not t.is_cuda or t.device != dev:
        raise ValueError(f"{name} must be on the CUDA device {dev} (no CPU fallback), got {t.device}")
    t = t.detach()
    if width is None:
        t = t.reshape(-1)
    elif t.dim() != 2 or t.shape[1] != width:
        raise ValueError(f"{name} must be [n, {width}], got {list(t.shape)}")
    return t.contiguous()


def _check_finite(tensors):
    """ValueError unless every element is finite: one 4-byte read back for all of them."""
    flags = torch.stack([torch.isfinite(t).all() for t in tensors if t is not None])
    if not bool(flags.all()):
        raise ValueError("frosting initialisation: an input is not finite")


def _gaussians(gaussians, dev):
    if not isinstance(gaussians, (tuple, list)) or len(gaussians) != 4:
        raise ValueError("gaussians must be the activated (points, scaling, quaternions, strengths)")
    points, scaling, quats, strengths = gaussians
    g = (_rows(points, "points", dev, 3), _rows(scaling, "scaling", dev, 3), _rows(quats, "quaternions", dev, 4),
         _rows(strengths, "strengths", dev, None))
    if not g[0].shape[0] == g[1].shape[0] == g[2].shape[0] == g[3].shape[0]:
        raise ValueError("points, scaling, quaternions and strengths need one row per Gaussian")
    return g


def _fractions(n_samples, dev):
    """torch.linspace(0, 1, n), as the reference samples: torch's linspace fills its two halves from either end."""
    return torch.linspace(0., 1., n_samples, device=dev)


def _extents(P, K, n_samples, smooth_K, V):
    if not 1 <= n_samples <= MAX_SAMPLES:
        raise ValueError(f"n_samples must be within [1, {MAX_SAMPLES}], got {n_samples}")
    if not 1 <= K <= 32 or K > P:
        raise ValueError(f"K must be within [1, 32] and at most the {P} Gaussians, got {K}")
    if not 0 <= smooth_K <= 32 or smooth_K > V:
        raise ValueError(f"smooth_K must be within [0, 32] and at most the {V} vertices, got {smooth_K}")


def _layer(min_layer_size, spatial_extent):
    """(min_layer_size * extent, 0.5 * min_layer_size * extent): Python floats, rounded to float32 where the reference's
    torch ops meet them; min_layer_size <= 0 turns the widening off."""
    if min_layer_size <= 0:
        return 0.0, 0.0
    return float(min_layer_size * spatial_extent), float(0.5 * min_layer_size * spatial_extent)


def _run(dev, verts, normals, g, knn_idx, inner_range, outer_range, n_samples, level, smooth_idx, layer,
         min_clamp_inner=None, max_clamp_outer=None, faces=None, std_idx=None, std_range=0.0, densities=None):
    V = verts.shape[0]
    o = dict(dtype=torch.float32, device=dev)
    level_outer, level_inner = torch.empty(V, **o), torch.empty(V, **o)
    out = LevelPoints(torch.empty(V, **o), torch.empty(V, **o), torch.empty(V, 3, **o), torch.empty(V, 3, **o))
    fr = _fractions(n_samples, dev)
    vf_offsets = vf_faces = None
    if faces is not None:
        flat = faces.long().reshape(-1)
        vf_faces = (torch.sort(flat, stable=True).indices // 3).to(torch.int32)      # faces ascending per vertex
        vf_offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev),
                                torch.bincount(flat, minlength=V).cumsum(0)]).to(torch.int32)
    points, scaling, quats, strengths = g
    st = _lib.FrostingInit(
        n_verts=V, n_faces=0 if faces is None else faces.shape[0], P=points.shape[0], K=knn_idx.shape[1],
        n_samples=n_samples, smooth_K=0 if smooth_idx is None else smooth_idx.shape[1],
        std_K=0 if std_idx is None else std_idx.shape[1], level=float(level), std_range=float(std_range),
        min_layer=layer[0], half_layer=layer[1], d_verts=ptr(verts), d_faces=ptr(faces), d_vf_offsets=ptr(vf_offsets),
        d_vf_faces=ptr(vf_faces), d_normals=ptr(normals), d_points=ptr(points), d_scaling=ptr(scaling),
        d_quaternions=ptr(quats), d_strengths=ptr(strengths), d_knn_idx=ptr(knn_idx), d_std_idx=ptr(std_idx),
        d_inner_range=ptr(inner_range), d_outer_range=ptr(outer_range), d_min_clamp_inner=ptr(min_clamp_inner),
        d_max_clamp_outer=ptr(max_clamp_outer), d_fractions=ptr(fr), d_smooth_idx=ptr(smooth_idx),
        d_level_outer=ptr(level_outer), d_level_inner=ptr(level_inner), d_outer_dist=ptr(out.outer_dist),
        d_inner_dist=ptr(out.inner_dist), d_outer_verts=ptr(out.outer_verts), d_inner_verts=ptr(out.inner_verts),
        d_densities=ptr(densities))
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fb200_level_points(C.byref(st), stream(dev)))
    return out


def level_points_along_normals(gaussians, verts, normals, inner_range, outer_range, *, n_samples=21, K=16, level,
                               smooth_K=4, min_layer_size=0., spatial_extent, min_clamp_inner=None,
                               max_clamp_outer=None, return_densities=False):
    """compute_level_points_along_normals (frosting_model.py:2016-2208, use_last_intersection_as_inner_level_point=True)
    on the GPU.  `gaussians` is the activated (points [P,3], scaling [P,3], quaternions [P,4], strengths [P] or [P,1]);
    verts, normals [V,3]; inner_range, outer_range, min_clamp_inner, max_clamp_outer [V]; all float32 on one CUDA
    device.  Returns LevelPoints(outer_dist [V], inner_dist [V], outer_verts [V,3], inner_verts [V,3]), and with
    `return_densities` also the [V, n_samples] sample densities.  ValueError on bad shapes, dtypes or devices, K > P,
    n_samples > 32 and non-finite inputs."""
    dev = verts.device if isinstance(verts, torch.Tensor) else None
    with torch.no_grad():
        verts = _rows(verts, "verts", dev, 3)
        V = verts.shape[0]
        normals = _rows(normals, "normals", dev, 3)
        g = _gaussians(gaussians, dev)
        ranges = [_rows(t, name, dev, None) for t, name in ((inner_range, "inner_range"), (outer_range, "outer_range"))]
        clamps = [None if t is None else _rows(t, name, dev, None)
                  for t, name in ((min_clamp_inner, "min_clamp_inner"), (max_clamp_outer, "max_clamp_outer"))]
        if normals.shape[0] != V or any(t is not None and t.numel() != V for t in ranges + clamps):
            raise ValueError("normals, ranges and clamps need one row per vertex")
        n_samples, K, smooth_K = int(n_samples), int(K), int(smooth_K)
        _extents(g[0].shape[0], K, n_samples, smooth_K, V)
        _check_finite([verts, normals, *g, *ranges, *clamps])
        knn_idx = knn_points(verts, g[0], K=K).idx
        smooth_idx = knn_points(verts, K=smooth_K).idx if smooth_K > 0 else None
        dens = torch.empty(V, n_samples, dtype=torch.float32, device=dev) if return_densities else None
        out = _run(dev, verts, normals, g, knn_idx, ranges[0], ranges[1], n_samples, level, smooth_idx,
                   _layer(min_layer_size, spatial_extent), clamps[0], clamps[1], densities=dens)
        return (out, dens) if return_densities else out


def initial_shell(sugar, gs, verts, faces, spatial_extent, *, n_samples=21, K=16, level=0.01, smooth_K=4,
                  min_frosting_size=0.001, initial_proposal_std_range=3., final_proposal_range=3.,
                  final_clamping_range=0.1):
    """Frosting.__init__'s thickness (frosting_model.py:296-369) with its defaults: the base mesh's vertex normals, the
    proposal from the SuGaR Gaussians `sugar` (+-initial_proposal_std_range times the mean width of the smooth_K
    nearest ones along the normal), then the level points of the 3DGS Gaussians `gs` inside the proposal widened by
    final_proposal_range and clamped to final_clamping_range of it.  `sugar` and `gs` are activated (points, scaling,
    quaternions, strengths); verts [V,3] float32 and faces [F,3] integer on one CUDA device.  Returns
    LevelPoints(outer_dist, inner_dist, outer_verts, inner_verts): Frosting's _outer_dist / _inner_dist and shell."""
    return _initial_shell(sugar, gs, verts, faces, spatial_extent, n_samples=n_samples, K=K, level=level,
                          smooth_K=smooth_K, min_frosting_size=min_frosting_size,
                          initial_proposal_std_range=initial_proposal_std_range,
                          final_proposal_range=final_proposal_range, final_clamping_range=final_clamping_range)[0]


def _faces(faces, dev, V):
    if not isinstance(faces, torch.Tensor) or faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point \
            or faces.device != dev:
        raise ValueError(f"faces must be an integer [F, 3] tensor on {dev}")
    faces = faces.to(torch.int32).contiguous()
    if faces.numel() and (int(faces.min()) < 0 or int(faces.max()) >= V):
        raise ValueError(f"faces must index the {V} vertices")
    return faces


def _initial_shell(sugar, gs, verts, faces, spatial_extent, *, n_samples, K, level, smooth_K, min_frosting_size,
                   initial_proposal_std_range, final_proposal_range, final_clamping_range):
    """initial_shell's LevelPoints and the base mesh's vertex normals [V,3] it computed on the way."""
    dev = verts.device if isinstance(verts, torch.Tensor) else None
    with torch.no_grad():
        verts = _rows(verts, "verts", dev, 3)
        V = verts.shape[0]
        faces = _faces(faces, dev, V)
        gs_s, gs_v = _gaussians(sugar, dev), _gaussians(gs, dev)
        n_samples, K, smooth_K = int(n_samples), int(K), int(smooth_K)
        _extents(min(gs_s[0].shape[0], gs_v[0].shape[0]), K, n_samples, smooth_K, V)
        if not 1 <= smooth_K <= gs_s[0].shape[0]:
            raise ValueError("the proposal averages over smooth_K >= 1 SuGaR Gaussians")
        _check_finite([verts, *gs_s, *gs_v])
        layer = _layer(min_frosting_size, spatial_extent)
        o = dict(dtype=torch.float32, device=dev)
        normals, inner_range, outer_range = torch.empty(V, 3, **o), torch.empty(V, **o), torch.empty(V, **o)
        std_idx = knn_points(verts, gs_s[0], K=smooth_K).idx
        smooth_idx = knn_points(verts, K=smooth_K).idx
        surface = _run(dev, verts, normals, gs_s, knn_points(verts, gs_s[0], K=K).idx, inner_range, outer_range,
                       n_samples, level, smooth_idx, layer, faces=faces, std_idx=std_idx,
                       std_range=initial_proposal_std_range)
        centre = (surface.outer_dist + surface.inner_dist) / 2
        min_outer = centre + final_proposal_range * (surface.outer_dist - centre)
        max_inner = centre + final_proposal_range * (surface.inner_dist - centre)
        clamp_outer = centre + final_clamping_range * (surface.outer_dist - centre)
        clamp_inner = centre + final_clamping_range * (surface.inner_dist - centre)
        return _run(dev, verts, normals, gs_v, knn_points(verts, gs_v[0], K=K).idx, max_inner, min_outer, n_samples,
                    level, smooth_idx, layer, clamp_inner, clamp_outer), normals


def torch_reference(gaussians, verts, normals, inner_range, outer_range, *, n_samples=21, K=16, level, smooth_K=4,
                    min_layer_size=0., spatial_extent, min_clamp_inner=None, max_clamp_outer=None, knn_idx,
                    smooth_idx=None, n_points_per_pass=2_000_000, return_densities=False):
    """compute_level_points_along_normals restated in torch for the dtype of its inputs, chunked over samples as the
    reference (frosting_model.py:2078-2200), with the neighbour tables given: knn_idx [V,K] into the Gaussians,
    smooth_idx [V,smooth_K] into the vertices.  pytorch3d's quaternion_to_matrix is scenes.quaternion_to_matrix."""
    from .scenes import quaternion_to_matrix
    xyz, scaling, rotation, strengths = gaussians
    strengths = strengths.reshape(-1, 1)
    dev, dt = verts.device, verts.dtype
    verts_range = torch.linspace(0., 1., n_samples, dtype=dt).to(dev).view(1, -1, 1)
    verts_range = verts_range * (inner_range - outer_range)[..., None, None] + outer_range[..., None, None]
    samples = (verts[:, None, :] + verts_range * normals[:, None, :]).view(-1, 3)
    samples_idx = knn_idx[:, None, :].expand(-1, n_samples, -1).reshape(-1, K)
    densities = torch.zeros(len(samples), dtype=dt, device=dev)
    inv_scaled_rotation = quaternion_to_matrix(rotation) * (1. / scaling.clamp(min=1e-8))[:, None]
    for i in range(0, len(samples), n_points_per_pass):
        j = min(len(samples), i + n_points_per_pass)
        idx = samples_idx[i:j]
        shift = samples[i:j, None] - xyz[idx]
        warped = inv_scaled_rotation[idx].transpose(-1, -2) @ shift[..., None]
        o = (warped[..., 0] * warped[..., 0]).sum(dim=-1).clamp(min=0., max=1e8)
        d = (strengths[idx][..., 0] * torch.exp(-1. / 2 * o)).sum(dim=-1)
        m = d >= 1.
        d[m] = d[m] / (d[m] + 1e-12)
        densities[i:j] = d
    densities = densities.reshape(-1, n_samples)
    under, above = densities - level < 0, densities - level > 0
    first = above.max(dim=-1, keepdim=True)[1]
    last = (n_samples - 1) - above.flip(dims=(-1,)).max(dim=-1, keepdim=True)[1]
    r = verts_range[..., 0]
    outer_dist = 0. + r[:, 0]
    ok = first[:, 0] > 0
    f = first[ok]
    v1, v0 = densities[ok].gather(-1, f).view(-1), densities[ok].gather(-1, f - 1).view(-1)
    t1, t0 = r[ok].gather(-1, f).view(-1), r[ok].gather(-1, f - 1).view(-1)
    outer_dist[ok] = (level - v0) / (v1 - v0) * (t1 - t0) + t0
    inner_dist = 0. + r[:, -1]
    ok_last = last[:, 0] < n_samples - 1
    lst = last[ok_last]
    vl, va = densities[ok_last].gather(-1, lst).view(-1), densities[ok_last].gather(-1, lst + 1).view(-1)
    tl, ta = r[ok_last].gather(-1, lst).view(-1), r[ok_last].gather(-1, lst + 1).view(-1)
    inner_dist[ok_last] = (level - vl) / (va - vl) * (ta - tl) + tl
    empty = (~ok) & (~ok_last) & under[:, 0]
    outer_dist[empty] = (inner_range + outer_range)[empty] / 2
    inner_dist[empty] = (inner_range + outer_range)[empty] / 2
    if min_layer_size > 0:
        flat = (inner_dist - outer_dist).abs() < min_layer_size * spatial_extent
        c = (inner_range + outer_range)[flat] / 2
        outer_dist[flat] = c - 0.5 * min_layer_size * spatial_extent
        inner_dist[flat] = c + 0.5 * min_layer_size * spatial_extent
    if min_clamp_inner is not None:
        inner_dist = inner_dist.clamp_min(min_clamp_inner)
    if max_clamp_outer is not None:
        outer_dist = outer_dist.clamp_max(max_clamp_outer)
    if smooth_idx is not None:
        outer_dist = outer_dist[smooth_idx].mean(dim=1)
        inner_dist = inner_dist[smooth_idx].mean(dim=1)
    out = LevelPoints(outer_dist, inner_dist, verts + outer_dist[:, None] * normals, verts + inner_dist[:, None] * normals)
    return (out, densities) if return_densities else out


def torch_initial_shell(sugar, gs, verts, faces, spatial_extent, *, n_samples=21, K=16, level=0.01, smooth_K=4,
                        min_frosting_size=0.001, initial_proposal_std_range=3., final_proposal_range=3.,
                        final_clamping_range=0.1, n_points_per_pass=2_000_000):
    """initial_shell restated in torch (frosting_model.py:296-369) for the dtype of its inputs, with pytorch3d's knn,
    normals and quaternion maths replaced by knn_points (tables computed in float32) and the scenes restatements."""
    from .scenes import p3d_verts_normals, quaternion_apply, quaternion_invert
    f32 = lambda t: t.float().contiguous()
    normals = p3d_verts_normals(verts, faces)
    std_idx = knn_points(f32(verts), f32(sugar[0]), K=smooth_K).idx
    smooth_idx = knn_points(f32(verts), K=smooth_K).idx
    stds = (sugar[1][std_idx] * quaternion_apply(quaternion_invert(sugar[2][std_idx]), normals[:, None])).norm(dim=-1)
    stds = stds.mean(dim=-1)
    common = dict(n_samples=n_samples, K=K, level=level, min_layer_size=min_frosting_size, spatial_extent=spatial_extent,
                  smooth_K=smooth_K, smooth_idx=smooth_idx, n_points_per_pass=n_points_per_pass)
    surface = torch_reference(sugar, verts, normals, initial_proposal_std_range * stds,
                              -1. * initial_proposal_std_range * stds,
                              knn_idx=knn_points(f32(verts), f32(sugar[0]), K=K).idx, **common)
    centre = (surface.outer_dist + surface.inner_dist) / 2
    return torch_reference(gs, verts, normals, centre + final_proposal_range * (surface.inner_dist - centre),
                           centre + final_proposal_range * (surface.outer_dist - centre),
                           min_clamp_inner=centre + final_clamping_range * (surface.inner_dist - centre),
                           max_clamp_outer=centre + final_clamping_range * (surface.outer_dist - centre),
                           knn_idx=knn_points(f32(verts), f32(gs[0]), K=K).idx, **common)
