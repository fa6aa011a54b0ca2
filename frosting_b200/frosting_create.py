"""A new Frosting layer from its thickness -- host side of the creation kernels of csrc/frosting_init.cu.

`Frosting.__init__` (frosting_scene/frosting_model.py:398-591) trims the shell so that it does not intersect itself,
samples the frosting Gaussians in its prism cells and splits off the background Gaussians.  Here, without pytorch3d and
without simple-knn:

    params, mesh = create_frosting((sugar.points, sugar.scaling, sugar.quaternions, sugar.strengths),
                                   {k: getattr(gaussians, k) for k in GS_KEYS}, verts, faces,
                                   spatial_extent=extent, camera_center=cameras.mean_centre)

`params` / `mesh` are the dicts `frosting_render` and `FrostingBlock` take.  The draws stay torch's
(`torch.multinomial`, then `torch.rand(N, 6)`, on the caller's generator), so a seeded run consumes the reference's
random stream; everything computed from them runs in the library.  `torch_trim_shell` and `torch_create_frosting`
restate the reference's torch computation for any dtype: the comparison routes of the tests and the benchmark.
"""
import ctypes as C
import math
from collections import namedtuple

import torch

from . import _lib
from ._lib import ptr, stream
from .frosting_init import _check_finite, _faces, _gaussians, _initial_shell, _rows
from .frosting_render import BG_KEYS
from .knn import knn_points

Trimmed = namedtuple("Trimmed", "inner_dist outer_dist inner_verts outer_verts inner_stop outer_stop")
# the raw parameters of a 3DGS GaussianModel create_frosting reads, as its attribute names
GS_KEYS = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")
SH_REST = 15                      # sh_levels = 4
THICKNESS = dict(n_samples=21, K=16, level=0.01, smooth_K=4, initial_proposal_std_range=3., final_proposal_range=3.,
                 final_clamping_range=0.1)


def _f32(x):
    """A Python float rounded to float32, as torch rounds a scalar operand of a float32 tensor op."""
    return float(torch.tensor(x, dtype=torch.float32))


def _struct(**kw):
    return _lib.FrostingCreate(**{k: (ptr(v) if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})


def _call(name, st, dev):
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), name)(C.byref(st), stream(dev)))


def _trim(verts, faces, normals, inner, outer, spatial_extent, n_iterations, proj_th):
    dev, V, F = verts.device, verts.shape[0], faces.shape[0]
    o = dict(dtype=torch.float32, device=dev)
    out = dict(d_inner_dist=torch.empty(V, **o), d_outer_dist=torch.empty(V, **o),
               d_inner_stop=torch.empty(V, dtype=torch.int32, device=dev),
               d_outer_stop=torch.empty(V, dtype=torch.int32, device=dev))
    nbytes = _lib.lib().fb200_knn_workspace_bytes(F, 2 * V, _lib.TRIM_K)
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
    ws = ws[(-ws.data_ptr()) % 256:]
    shell, centres = torch.empty(2 * V, 3, **o), torch.empty(F, 3, **o)
    knn_d, knn_i = torch.empty(2 * V, _lib.TRIM_K, **o), torch.empty(2 * V, _lib.TRIM_K, dtype=torch.int64, device=dev)
    st = _struct(n_verts=V, n_faces=F, n_iterations=n_iterations, step=_f32(1 / n_iterations),
                 inside_th=_f32(spatial_extent * proj_th), d_verts=verts, d_faces=faces, d_normals=normals,
                 d_inner_init=inner, d_outer_init=outer, d_shell=shell, d_centres=centres, d_knn_workspace=ws,
                 knn_workspace_bytes=nbytes, d_knn_dists=knn_d, d_knn_idx=knn_i, **out)
    _call("fb200_frosting_trim", st, dev)
    i, o_ = out["d_inner_dist"], out["d_outer_dist"]
    # the model's shell: Frosting.inner_verts / outer_verts over the trimmed distances
    return Trimmed(i, o_, verts + i[:, None] * normals, verts + o_[:, None] * normals, out["d_inner_stop"],
                   out["d_outer_stop"]), dict(shell=shell, centres=centres, knn_idx=knn_i)


def _check_trim(V, F, n_iterations, k):
    if k != _lib.TRIM_K:
        raise ValueError(f"k must be {_lib.TRIM_K}, the neighbour count Frosting trims with")
    if int(n_iterations) < 1:
        raise ValueError("n_iterations must be >= 1")
    if V > 0 and F < _lib.TRIM_K:
        raise ValueError(f"trimming tests the {_lib.TRIM_K} nearest cells: it needs at least {_lib.TRIM_K} faces, got {F}")


def trim_shell(verts, faces, normals, inner_dist, outer_dist, spatial_extent, *, n_iterations=20, k=8, proj_th=1e-6):
    """Frosting.__init__'s self-intersection trimming (frosting_model.py:398-435, is_inside_frosting :1675-1737) on the
    GPU.  verts, normals [V,3] and the untrimmed inner_dist, outer_dist [V] float32, faces [F,3] integer, on one CUDA
    device.  Returns Trimmed(inner_dist, outer_dist, inner_verts, outer_verts, inner_stop, outer_stop): the trimmed
    distances and shell, and per vertex side the iteration at which it stopped growing (n_iterations: never)."""
    dev = verts.device if isinstance(verts, torch.Tensor) else None
    with torch.no_grad():
        verts = _rows(verts, "verts", dev, 3)
        V = verts.shape[0]
        faces = _faces(faces, dev, V)
        normals = _rows(normals, "normals", dev, 3)
        inner, outer = _rows(inner_dist, "inner_dist", dev, None), _rows(outer_dist, "outer_dist", dev, None)
        if normals.shape[0] != V or inner.numel() != V or outer.numel() != V:
            raise ValueError("normals and distances need one row per vertex")
        _check_trim(V, faces.shape[0], n_iterations, k)
        _check_finite([verts, normals, inner, outer])
        return _trim(verts, faces, normals, inner, outer, spatial_extent, int(n_iterations), proj_th)[0]


def cell_counts(n_faces, n_gaussians, n_min_per_cell="auto"):
    """(n_min, N): Frosting's minimum per cell (ceil(N / 2F) for 'auto') and its number of Gaussians, raised to
    F * n_min when that is larger (frosting_model.py:476-484)."""
    if n_min_per_cell == "auto":
        n_min_per_cell = int(math.ceil(n_gaussians / (2 * n_faces)))
    n_min_per_cell = int(n_min_per_cell)
    return n_min_per_cell, max(int(n_gaussians), n_faces * n_min_per_cell)


def _draw_cells(volumes, n_min, N, generator):
    F = volumes.shape[0]
    cells = torch.arange(F, device=volumes.device).repeat(n_min)
    if N > F * n_min:
        extra = torch.multinomial(volumes / volumes.sum(), N - F * n_min, replacement=True, generator=generator)
        cells = torch.cat([cells, extra])
    return cells


def _gs(gs, dev):
    if not isinstance(gs, dict) or any(k not in gs for k in GS_KEYS):
        raise ValueError(f"gs must map each of {GS_KEYS} to the 3DGS model's raw parameter")
    xyz = _rows(gs["_xyz"], "gs _xyz", dev, 3)
    P = xyz.shape[0]
    t = dict(_xyz=xyz, _scaling=_rows(gs["_scaling"], "gs _scaling", dev, 3),
             _rotation=_rows(gs["_rotation"], "gs _rotation", dev, 4), _opacity=_rows(gs["_opacity"], "gs _opacity",
                                                                                     dev, None))
    for k, rows in (("_features_dc", 1), ("_features_rest", SH_REST)):
        f = gs[k]
        if not isinstance(f, torch.Tensor) or f.dim() != 3 or f.shape[1:] != (rows, 3):
            raise ValueError(f"gs {k} must be [P, {rows}, 3] (sh_levels = 4), got "
                             f"{list(f.shape) if isinstance(f, torch.Tensor) else type(f).__name__}")
        t[k] = _rows(f.reshape(f.shape[0], -1), f"gs {k}", dev, 3 * rows).view(-1, rows, 3)
    if any(v.shape[0] != P for v in t.values()):
        raise ValueError("the 3DGS parameters need one row per Gaussian")
    return t


def gs_activated(gs):
    """(get_xyz, get_scaling, get_rotation, get_opacity) of a 3DGS GaussianModel from its raw parameters."""
    return (gs["_xyz"], torch.exp(gs["_scaling"]), torch.nn.functional.normalize(gs["_rotation"]),
            torch.sigmoid(gs["_opacity"]).reshape(-1, 1))


def _background(gs, verts):
    """The 3DGS Gaussians not strictly inside the base vertices' bounding box, raw, in order (frosting_model.py:564-591)."""
    lo, hi = verts.min(dim=0, keepdim=True)[0], verts.max(dim=0, keepdim=True)[0]
    bg = ~((gs["_xyz"] > lo).all(dim=-1) & (gs["_xyz"] < hi).all(dim=-1))
    return dict(bg_points=gs["_xyz"][bg], bg_opacity_logits=gs["_opacity"].reshape(-1)[bg],
                bg_log_scales=gs["_scaling"][bg], bg_quats=gs["_rotation"][bg], bg_sh_dc=gs["_features_dc"][bg],
                bg_sh_rest=gs["_features_rest"][bg])


def create_frosting(sugar, gs, verts, faces, *, spatial_extent, camera_center, n_gaussians=2_000_000,
                    n_min_per_cell="auto", generator=None, avoid_self_intersections=True, contract_points=True,
                    use_background_gaussians=True, min_frosting_size=0.001):
    """Frosting.__init__ (frosting_model.py:296-591) with its defaults, from the coarse SuGaR model `sugar` (activated
    points, scaling, quaternions, strengths), the 3DGS model's raw parameters `gs` (GS_KEYS; sh_levels = 4), the base
    mesh verts [V,3] float32 / faces [F,3] integer, the training cameras' spatial extent and mean camera centre [3], all
    on one CUDA device.  Returns (params, mesh): MESH_KEYS and, where any 3DGS Gaussian lies outside the base mesh's
    bounding box, BG_KEYS; mesh = dict(verts, faces, inner, outer, cells) with the trimmed shell.  Draws with
    `generator` (None: the device's default).  ValueError on bad dtypes, devices or shapes, fewer than 8 faces when
    trimming, fewer than 4 frosting Gaussians and non-finite inputs."""
    return _create(sugar, gs, verts, faces, spatial_extent=spatial_extent, camera_center=camera_center,
                   n_gaussians=n_gaussians, n_min_per_cell=n_min_per_cell, generator=generator,
                   avoid_self_intersections=avoid_self_intersections, contract_points=contract_points,
                   use_background_gaussians=use_background_gaussians, min_frosting_size=min_frosting_size)[:2]


def _create(sugar, gs, verts, faces, *, spatial_extent, camera_center, n_gaussians=2_000_000, n_min_per_cell="auto",
            generator=None, avoid_self_intersections=True, contract_points=True, use_background_gaussians=True,
            min_frosting_size=0.001):
    """create_frosting's (params, mesh) and its intermediate values by name."""
    dev = verts.device if isinstance(verts, torch.Tensor) else None
    with torch.no_grad():
        verts = _rows(verts, "verts", dev, 3)
        V = verts.shape[0]
        faces = _faces(faces, dev, V)
        F = faces.shape[0]
        sug, g = _gaussians(sugar, dev), _gs(gs, dev)
        centre = _rows(camera_center, "camera_center", dev, None)
        if centre.numel() != 3:
            raise ValueError("camera_center must hold 3 coordinates")
        if not spatial_extent > 0:
            raise ValueError("spatial_extent must be > 0")
        if F < 1:
            raise ValueError("the base mesh needs faces")
        if avoid_self_intersections:
            _check_trim(V, F, 20, _lib.TRIM_K)
        n_min, N = cell_counts(F, n_gaussians, n_min_per_cell)
        if N < 4:
            raise ValueError(f"distCUDA2's scales need at least 4 frosting Gaussians, got {N}")
        _check_finite([verts, *sug, *g.values(), centre])
        lp, normals = _initial_shell(sug, gs_activated(g), verts, faces, spatial_extent,
                                     min_frosting_size=min_frosting_size, **THICKNESS)
        info = dict(thickness=lp, normals=normals)
        if avoid_self_intersections:
            trimmed, info["trim"] = _trim(verts, faces, normals, lp.inner_dist, lp.outer_dist, spatial_extent, 20, 1e-6)
            inner, outer, shell = trimmed.inner_dist, trimmed.outer_dist, (trimmed.inner_verts, trimmed.outer_verts)
            info["trimmed"] = trimmed
        else:
            inner, outer, shell = lp.inner_dist, lp.outer_dist, (lp.inner_verts, lp.outer_verts)
        o = dict(dtype=torch.float32, device=dev)
        common = dict(n_verts=V, n_faces=F, n_iterations=1, n_gaussians=N, n_gs=g["_xyz"].shape[0], sh_rest=SH_REST,
                      contract=int(bool(contract_points)), extent=_f32(spatial_extent),
                      min_height=_f32(min_frosting_size * spatial_extent), d_verts=verts, d_faces=faces)
        volumes = torch.empty(F, **o)
        _call("fb200_frosting_volumes", _struct(d_inner_dist=inner, d_outer_dist=outer, d_camera_center=centre,
                                                d_volumes=volumes, **common), dev)
        cells = _draw_cells(volumes, n_min, N, generator)
        u = torch.rand(N, 6, device=dev, generator=generator)
        p = dict(bary_logits=torch.empty(N, 6, **o), points=torch.empty(N, 3, **o), max_scales=torch.empty(N, **o))
        _call("fb200_frosting_sample", _struct(d_inner_verts=lp.inner_verts, d_outer_verts=lp.outer_verts, d_cells=cells,
                                               d_u=u, **{"d_" + k: v for k, v in p.items()}, **common), dev)
        nn_idx = knn_points(p["points"], K=4).idx
        sh_idx = knn_points(p["points"], g["_xyz"], K=1).idx.reshape(-1)
        out = dict(dist2=torch.empty(N, **o), log_scales=torch.empty(N, 3, **o), quats=torch.empty(N, 4, **o),
                   opacity_logits=torch.empty(N, **o), sh_dc=torch.empty(N, 1, 3, **o),
                   sh_rest=torch.empty(N, SH_REST, 3, **o))
        _call("fb200_frosting_finish", _struct(d_points=p["points"], d_max_scales=p["max_scales"], d_nn_idx=nn_idx,
                                               d_sh_idx=sh_idx, d_gs_sh_dc=g["_features_dc"],
                                               d_gs_sh_rest=g["_features_rest"], **{"d_" + k: v for k, v in out.items()},
                                               **common), dev)
        params = dict(bary_logits=p["bary_logits"], opacity_logits=out["opacity_logits"], log_scales=out["log_scales"],
                      quats=out["quats"], sh_dc=out["sh_dc"], sh_rest=out["sh_rest"])
        if use_background_gaussians:
            bg = _background(g, verts)
            if bg["bg_points"].shape[0] > 0:
                params.update({k: bg[k].contiguous() for k in BG_KEYS})
        mesh = dict(verts=verts, faces=faces, inner=shell[0], outer=shell[1], cells=cells)
        info.update(volumes=volumes, u=u, n_min=n_min, points=p["points"], max_scales=p["max_scales"], nn_idx=nn_idx,
                    sh_idx=sh_idx, dist2=out["dist2"])
        return params, mesh, info


# ---------------------------------------------------------------------------------------------------------------------
# The reference's torch computation, for any dtype, with the neighbour tables from `knn(queries, points, K) -> idx`
# (default: knn_points over float32 copies)

def _knn32(queries, points, K):
    return knn_points(queries.float().contiguous(), points.float().contiguous(), K=K).idx


def _is_inside(cells, points, spatial_extent, k, proj_th, knn):
    """is_inside_frosting (frosting_model.py:1675-1737) over the cells [F,2,3,3]."""
    nrm = torch.nn.functional.normalize
    cv = cells
    normals = torch.cat([
        nrm(torch.cross(cv[:, 0, 1] - cv[:, 0, 0], cv[:, 1, 0] - cv[:, 0, 0], dim=-1), dim=-1)[:, None],
        nrm(torch.cross(cv[:, 0, 2] - cv[:, 0, 1], cv[:, 1, 1] - cv[:, 0, 1], dim=-1), dim=-1)[:, None],
        nrm(torch.cross(cv[:, 1, 0] - cv[:, 0, 0], cv[:, 0, 2] - cv[:, 0, 0], dim=-1), dim=-1)[:, None],
        nrm(torch.cross(cv[:, 0, 2] - cv[:, 0, 0], cv[:, 0, 1] - cv[:, 0, 0], dim=-1), dim=-1)[:, None],
        nrm(torch.cross(cv[:, 1, 1] - cv[:, 1, 0], cv[:, 1, 2] - cv[:, 1, 0], dim=-1), dim=-1)[:, None]], dim=1)
    face_points = torch.cat([cv[:, 0, 0][:, None], cv[:, 0, 1][:, None], cv[:, 0, 0][:, None], cv[:, 0, 0][:, None],
                             cv[:, 1, 0][:, None]], dim=1)
    centres = cells.reshape(-1, 6, 3).mean(dim=1)
    idx = knn(points, centres, k)
    proj = ((points[:, None, None] - face_points[idx]) * normals[idx]).sum(dim=-1)
    return (proj > spatial_extent * proj_th).all(dim=-1).any(dim=-1)


def _cells(faces, inner_verts, outer_verts):
    return torch.cat([inner_verts[:, None], outer_verts[:, None]], dim=1)[faces.long()].transpose(-2, -3)


def torch_trim_shell(verts, faces, normals, inner_dist, outer_dist, spatial_extent, *, n_iterations=20, k=8,
                     proj_th=1e-6, knn=_knn32):
    """trim_shell restated with the reference's torch ops (frosting_model.py:398-435) for the dtype of its inputs."""
    old_inner, old_outer = inner_dist.clone(), outer_dist.clone()
    inner, outer = torch.zeros_like(inner_dist), torch.zeros_like(outer_dist)
    inner_mask = torch.ones_like(inner, dtype=torch.bool)
    outer_mask = torch.ones_like(outer, dtype=torch.bool)
    inner_stop = torch.full_like(inner, n_iterations, dtype=torch.int32)
    outer_stop = torch.full_like(outer, n_iterations, dtype=torch.int32)
    for it in range(n_iterations):
        inner_i, outer_i = inner.clone(), outer.clone()
        new_inner = inner_i[inner_mask] + 1 / n_iterations * old_inner[inner_mask]
        new_outer = outer_i[outer_mask] + 1 / n_iterations * old_outer[outer_mask]
        inner[inner_mask] = new_inner.clone()
        outer[outer_mask] = new_outer.clone()
        inner_verts, outer_verts = verts + inner[:, None] * normals, verts + outer[:, None] * normals
        cells = _cells(faces, inner_verts, outer_verts)
        inner_in = _is_inside(cells, inner_verts[inner_mask].clone(), spatial_extent, k, proj_th, knn)
        outer_in = _is_inside(cells, outer_verts[outer_mask].clone(), spatial_extent, k, proj_th, knn)
        new_inner[inner_in] = inner_i[inner_mask][inner_in]
        new_outer[outer_in] = outer_i[outer_mask][outer_in]
        inner[inner_mask] = new_inner.clone()
        outer[outer_mask] = new_outer.clone()
        inner_stop[inner_mask.nonzero()[:, 0][inner_in]] = it
        outer_stop[outer_mask.nonzero()[:, 0][outer_in]] = it
        inner_mask[inner_mask.clone()] = ~inner_in
        outer_mask[outer_mask.clone()] = ~outer_in
    return Trimmed(inner, outer, verts + inner[:, None] * normals, verts + outer[:, None] * normals, inner_stop,
                   outer_stop)


def _contract(x, c, L):
    res = x + 0.
    dists = (x - c).norm(dim=-1, keepdim=True)
    mask = dists[..., 0] > L
    res[mask] = c + L * (2 - L / dists[mask]) * ((x - c)[mask] / dists[mask])
    return res


def torch_cell_volumes(verts, faces, inner_dist, outer_dist, spatial_extent, camera_center, *, contract_points=True,
                       min_frosting_size=0.001):
    """The prism cell volumes of frosting_model.py:441-472."""
    fl = faces.long()
    fv = verts[fl]
    c = camera_center.reshape(1, 3)
    if contract_points:
        fv = _contract(fv.view(-1, 3), c, spatial_extent).view(-1, 3, 3)
    a = (fv[:, 0] - fv[:, 1]).norm(dim=-1)
    b = (fv[:, 1] - fv[:, 2]).norm(dim=-1)
    e = (fv[:, 2] - fv[:, 0]).norm(dim=-1)
    s = (a + b + e) / 2
    areas = (s * (s - a) * (s - b) * (s - e)).clamp_min(0.).sqrt()
    heights = (inner_dist - outer_dist).abs()
    heights.clamp_min_(min_frosting_size * spatial_extent)
    if contract_points:
        dists = (verts - c).norm(dim=-1)
        mask = dists > spatial_extent
        heights[mask] = heights[mask] * (spatial_extent / dists[mask]) ** 2
    return areas * heights[fl].mean(dim=-1)


def torch_sample(faces, inner_verts, outer_verts, cells, u, gs, knn=_knn32):
    """The frosting Gaussians of frosting_model.py:499-554 from the cell indices and the uniforms u [N,6]: dict of
    bary_logits, points, max_scales, dist2, log_scales, quats, opacity_logits, sh_dc, sh_rest."""
    cell_verts = _cells(faces, inner_verts, outer_verts)
    bary = u.clone()
    bary[..., -1] = 1.
    bary = bary.sort(dim=-1)[0]
    bary[..., 1:] = bary[..., 1:] - bary[..., :-1]
    points = (bary[..., None] * cell_verts[cells].reshape(-1, 6, 3)).sum(dim=-2)
    sides = (cell_verts[:, 1] - cell_verts[:, 0]).norm(dim=-1)
    bases = (cell_verts - cell_verts[:, :, [1, 2, 0]]).norm(dim=-1)
    max_scales = torch.cat([sides, bases.view(-1, 6)], dim=1).max(dim=-1)[0][cells]
    idx = knn(points, points, 4)[:, 1:]
    dist2 = ((points[idx] - points[:, None]) ** 2).sum(-1).sort(dim=-1)[0].mean(dim=-1)       # distCUDA2
    scales = torch.clamp_min(dist2.clamp_max(max_scales ** 2), 0.0000001).sqrt()
    nearest = knn(points, gs["_xyz"], 1)[:, 0]
    n = len(points)
    x = 0.1 * torch.ones(n, dtype=torch.float32, device=points.device)
    return dict(bary_logits=torch.log(bary.clamp_min(1e-8)), points=points, max_scales=max_scales, dist2=dist2,
                log_scales=torch.log(scales)[..., None].repeat(1, 3),
                quats=torch.tensor([1., 0., 0., 0.], dtype=points.dtype, device=points.device).repeat(n, 1),
                opacity_logits=torch.log(x / (1 - x)),     # inverse_sigmoid, float32 as the reference's
                sh_dc=gs["_features_dc"][nearest].clone(), sh_rest=gs["_features_rest"][nearest].clone())


def torch_create_frosting(sugar, gs, verts, faces, *, spatial_extent, camera_center, n_gaussians=2_000_000,
                          n_min_per_cell="auto", generator=None, avoid_self_intersections=True, contract_points=True,
                          use_background_gaussians=True, min_frosting_size=0.001, knn=_knn32):
    """create_frosting restated in the reference's torch ops for the dtype of its inputs: torch_initial_shell, then
    torch_trim_shell, the cell volumes, the draws and torch_sample; returns (params, mesh, volumes)."""
    from .frosting_init import torch_initial_shell
    from .scenes import p3d_verts_normals
    dev = verts.device
    normals = p3d_verts_normals(verts, faces)
    lp = torch_initial_shell(sugar, gs_activated(gs), verts, faces, spatial_extent, min_frosting_size=min_frosting_size,
                             **THICKNESS)
    inner, outer, shell = lp.inner_dist, lp.outer_dist, (lp.inner_verts, lp.outer_verts)
    if avoid_self_intersections:
        t = torch_trim_shell(verts, faces, normals, lp.inner_dist, lp.outer_dist, spatial_extent, knn=knn)
        inner, outer, shell = t.inner_dist, t.outer_dist, (t.inner_verts, t.outer_verts)
    volumes = torch_cell_volumes(verts, faces, inner, outer, spatial_extent, camera_center,
                                 contract_points=contract_points, min_frosting_size=min_frosting_size)
    n_min, N = cell_counts(len(faces), n_gaussians, n_min_per_cell)
    cells = _draw_cells(volumes, n_min, N, generator)
    u = torch.rand(N, 6, device=dev, generator=generator).to(verts.dtype)
    s = torch_sample(faces, lp.inner_verts, lp.outer_verts, cells, u, gs, knn)
    params = {k: s[k] for k in ("bary_logits", "opacity_logits", "log_scales", "quats", "sh_dc", "sh_rest")}
    if use_background_gaussians:
        bg = _background(gs, verts)
        if len(bg["bg_points"]):
            params.update(bg)
    return params, dict(verts=verts, faces=faces, inner=shell[0], outer=shell[1], cells=cells), volumes
