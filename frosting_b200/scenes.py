"""Synthetic cameras and scenes for tests and bench.py (SURVEY.md section 8d, BASELINE.md section 4).

Camera conventions restate the reference so that the same tensors can be fed to both rasterizers:
  getProjectionMatrix   frosting_utils/graphics_utils.py:65-85
  getWorld2View         frosting_utils/graphics_utils.py:38-50
  GSCamera matrices     frosting_scene/cameras.py:203-212 (world_view_transform = W2C^T,
                        full_proj_transform = world_view_transform @ P^T, camera_center = inv(W2C^T)[3,:3])
Frosting's mesh-bound parameterisation restates frosting_scene/frosting_model.py:
  prism cells           :676,705,709-710 (shell_cells_verts: inner v0..v2, outer v0..v2)
  points                :713-726 (softmax of 6 barycentric logits x cell vertices)
  activations           :729-734,765,798
  cell assignment       :476-495, barycentric init :503-509
Everything is generated on the CPU with a seeded torch.Generator (bit-reproducible across boxes) and
moved to the requested device.
"""
import math
from types import SimpleNamespace

import torch

from .rasterizer import GaussianRasterizationSettings

ZNEAR, ZFAR = 0.01, 100.0


def get_projection_matrix(znear, zfar, fovX, fovY):
    tan_y, tan_x = math.tan(fovY / 2), math.tan(fovX / 2)
    top, right = tan_y * znear, tan_x * znear
    bottom, left = -top, -right
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def make_camera(W, H, w2c=None, fovx_deg=60.0, device="cpu"):
    """GSCamera-like namespace.  w2c: 4x4 world-to-camera (COLMAP axes: x right, y down, z forward)."""
    if w2c is None:
        w2c = torch.eye(4)
    w2c = w2c.float()
    tanfovx = math.tan(math.radians(fovx_deg) / 2)
    tanfovy = tanfovx * H / W
    fovx, fovy = 2 * math.atan(tanfovx), 2 * math.atan(tanfovy)
    world_view = w2c.t().contiguous()
    proj = get_projection_matrix(ZNEAR, ZFAR, fovx, fovy).t().contiguous()
    full = world_view @ proj
    campos = torch.linalg.inv(world_view)[3, :3].contiguous()
    return SimpleNamespace(
        image_width=W, image_height=H, tanfovx=tanfovx, tanfovy=tanfovy, FoVx=fovx, FoVy=fovy,
        world_view_transform=world_view.to(device), projection_matrix=proj.to(device),
        full_proj_transform=full.to(device), camera_center=campos.to(device), w2c=w2c)


def look_at_w2c(eye, target, up=(0.0, -1.0, 0.0)):
    """World-to-camera for a camera at `eye` looking at `target` (z forward, y down)."""
    eye = torch.tensor(eye, dtype=torch.float64)
    target = torch.tensor(target, dtype=torch.float64)
    upv = torch.tensor(up, dtype=torch.float64)
    z = target - eye
    z = z / z.norm()
    x = torch.linalg.cross(-upv, z)     # right
    if x.norm() < 1e-8:
        x = torch.tensor([1.0, 0.0, 0.0], dtype=torch.float64)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)        # down
    R = torch.stack([x, y, z])          # rows: camera axes in world
    w2c = torch.eye(4, dtype=torch.float64)
    w2c[:3, :3] = R
    w2c[:3, 3] = -R @ eye
    return w2c.float()


def ring_cameras(n, W, H, centre=(0.0, 0.0, 6.0), radius=6.0, device="cpu"):
    cams = []
    for i in range(n):
        a = 2 * math.pi * i / n
        eye = (centre[0] + radius * math.sin(a), centre[1], centre[2] - radius * math.cos(a))
        cams.append(make_camera(W, H, look_at_w2c(eye, centre), device=device))
    return cams


def settings_for(cam, sh_degree, bg=None, device=None, scale_modifier=1.0, debug=False):
    device = device or cam.world_view_transform.device
    if bg is None:
        bg = torch.zeros(3)
    return GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width),
        tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg.float().to(device), scale_modifier=scale_modifier,
        viewmatrix=cam.world_view_transform.to(device), projmatrix=cam.full_proj_transform.to(device),
        sh_degree=sh_degree, campos=cam.camera_center.to(device), prefiltered=False, debug=debug)


def random_gaussians(P, cam, seed, device="cpu", sh_coeffs=16, large_frac=0.005, near_frac=0.02):
    """Free Gaussians in the frustum of `cam` (identity W2C assumed): SURVEY.md 8d recipe."""
    g = torch.Generator().manual_seed(seed)
    W = cam.image_width
    fx = W / (2 * cam.tanfovx)
    z = torch.rand(P, generator=g) * 8 + 2
    n_near = int(P * near_frac)
    if n_near:
        z[:n_near] = torch.rand(n_near, generator=g) * 1.2 - 1.0
    x = (torch.rand(P, generator=g) * 2 - 1) * 1.1 * z.abs() * cam.tanfovx
    y = (torch.rand(P, generator=g) * 2 - 1) * 1.1 * z.abs() * cam.tanfovy
    means = torch.stack([x, y, z], 1)
    # move into world space if the camera is not at the origin
    c2w = torch.linalg.inv(cam.w2c.double())
    means = (torch.cat([means.double(), torch.ones(P, 1, dtype=torch.float64)], 1) @ c2w.t())[:, :3].float()
    z_med = 6.0
    s0 = 1.5 * z_med / fx
    scales = s0 * torch.exp(0.5 * torch.randn(P, 3, generator=g))
    n_large = int(P * large_frac)
    if n_large:
        idx = torch.randperm(P, generator=g)[:n_large]
        scales[idx] *= 20
    q = torch.randn(P, 4, generator=g)
    rotations = q / q.norm(dim=1, keepdim=True)
    opacities = torch.rand(P, 1, generator=g) * 0.9 + 0.05
    shs = torch.randn(P, sh_coeffs, 3, generator=g) * 0.1
    shs[:, 0] = torch.randn(P, 3, generator=g)
    out = dict(means3D=means, scales=scales, rotations=rotations, opacities=opacities, shs=shs)
    return {k: v.contiguous().to(device) for k, v in out.items()}


def uv_sphere(n_lat, n_lon, radius=3.0, centre=(0.0, 0.0, 6.0)):
    """Closed UV sphere: 2 + (n_lat-1)*n_lon vertices, 2*n_lon*(n_lat-1) faces."""
    th = torch.linspace(0, math.pi, n_lat + 1)[1:-1]                    # polar, without the poles
    ph = torch.arange(n_lon) * (2 * math.pi / n_lon)
    st, ct = torch.sin(th)[:, None], torch.cos(th)[:, None]
    ring = torch.stack([st * torch.cos(ph)[None], ct.expand(-1, n_lon), st * torch.sin(ph)[None]], -1)  # [n_lat-1,n_lon,3]
    normals = torch.cat([torch.tensor([[0.0, 1.0, 0.0]]), ring.reshape(-1, 3), torch.tensor([[0.0, -1.0, 0.0]])])
    verts = normals * radius + torch.tensor(centre)
    nr = n_lat - 1

    def vid(i, j):
        return 1 + i * n_lon + (j % n_lon)
    j = torch.arange(n_lon)
    faces = []
    top = torch.stack([torch.zeros(n_lon, dtype=torch.long), 1 + (j + 1) % n_lon, 1 + j], 1)
    faces.append(top)
    for i in range(nr - 1):
        a, b = vid(i, j), vid(i, j + 1)
        c, d = vid(i + 1, j), vid(i + 1, j + 1)
        faces.append(torch.stack([a, b, d], 1))
        faces.append(torch.stack([a, d, c], 1))
    last = 1 + nr * n_lon
    bot = torch.stack([torch.full((n_lon,), last, dtype=torch.long), vid(nr - 1, j), vid(nr - 1, j + 1)], 1)
    faces.append(bot)
    return verts.float().contiguous(), torch.cat(faces).int().contiguous(), normals.float().contiguous()


def frosting_layer(P, cam, seed, n_faces_target=1_000_000, device="cpu", sh_coeffs=16, thickness=0.02,
                   n_min_per_cell=1, view_distance=7.5, n_background=0, behind_frac=0.25):
    """Frosting-layer scene: Gaussians bound to prism cells over a UV-sphere base mesh.

    Returns the *learnable parameters* (bary logits, opacity logits, log scales, raw quaternions, SH dc/rest)
    plus the mesh and `_point_cell_indices`; `frosting_attributes()` turns them into rasterizer inputs.
    `n_background` > 0 adds Frosting's background Gaussians (the six `bg_*` keys, frosting_model.py:564-591): free
    Gaussians outside the base mesh's bounding box, on a thick spherical shell around the scene, `behind_frac` of them
    behind the ring cameras (radius 6 around the sphere's centre); `frosting_background_attributes()` maps them.  They
    come from a generator of their own, so the mesh-bound tensors are the same with or without them.
    """
    g = torch.Generator().manual_seed(seed)
    n_lon = max(8, int(round(math.sqrt(n_faces_target / 2.0) * math.sqrt(2.0))))
    n_lat = max(4, n_faces_target // (2 * n_lon) + 1)
    verts, faces, normals = uv_sphere(n_lat, n_lon)
    F = faces.shape[0]
    inner = verts - thickness * normals
    outer = verts + thickness * normals
    fl = faces.long()
    # cell volumes ~ base triangle area (constant thickness)
    tri = verts[fl]
    area = torch.linalg.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]).norm(dim=1) * 0.5
    base = torch.arange(F).repeat(n_min_per_cell)[:P]
    n_extra = P - base.shape[0]
    if n_extra > 0:
        extra = torch.multinomial(area / area.sum(), n_extra, replacement=True, generator=g)
        cells = torch.cat([base, extra])
    else:
        cells = base
    # barycentric init: spacings of sorted uniforms (uniform on the simplex), stored as logits
    u = torch.sort(torch.rand(P, 5, generator=g), dim=1).values
    u = torch.cat([torch.zeros(P, 1), u, torch.ones(P, 1)], 1)
    bary = (u[:, 1:] - u[:, :-1]).clamp_min(1e-6)
    bary_logits = bary.log()
    fx = cam.image_width / (2 * cam.tanfovx)
    s0 = 1.5 * view_distance / fx     # median screen-space sigma ~1.5 px at the viewing distance
    log_scales = math.log(s0) + 0.5 * torch.randn(P, 3, generator=g)
    log_scales[:, 2] -= 1.0    # flatter along one axis, like surface-aligned splats
    quats = torch.randn(P, 4, generator=g)
    opacity_logits = torch.logit(torch.rand(P, generator=g) * 0.9 + 0.05)
    sh_dc = torch.randn(P, 1, 3, generator=g)
    sh_rest = torch.randn(P, sh_coeffs - 1, 3, generator=g) * 0.1
    params = dict(bary_logits=bary_logits, opacity_logits=opacity_logits, log_scales=log_scales, quats=quats,
                  sh_dc=sh_dc, sh_rest=sh_rest)
    mesh = dict(verts=verts, faces=faces, inner=inner, outer=outer, cells=cells)
    if n_background > 0:
        params.update(_background_gaussians(n_background, verts, fx, seed, sh_coeffs, behind_frac))
    params = {k: v.contiguous().to(device) for k, v in params.items()}
    mesh = {k: v.contiguous().to(device) for k, v in mesh.items()}
    return params, mesh


def _background_gaussians(n, verts, fx, seed, sh_coeffs, behind_frac):
    g = torch.Generator().manual_seed(seed + 0x6267)           # separate stream: the mesh-bound draws are unchanged
    lo, hi = verts.min(0).values, verts.max(0).values
    centre, half = (lo + hi) / 2, (hi - lo) / 2
    n_behind = int(n * behind_frac)
    d = torch.randn(n, 3, generator=g)
    d[:, 1] *= 0.5                                                # flatter towards the ring's plane
    d = d / d.norm(dim=1, keepdim=True)
    # distance along d at which the ray leaves the bounding box: beyond it a point is background (frosting_model.py:567-574)
    t_box = (half[None] / d.abs().clamp_min(1e-6)).min(1).values * 1.05
    # a thick shell: in front of the ring cameras (between the box and radius 5.5, the ring being at 6) or behind them
    u = torch.rand(n, generator=g)
    r = t_box + u * (5.5 - t_box).clamp_min(0.0)
    r[:n_behind] = torch.maximum(t_box[:n_behind], 7.0 + u[:n_behind] * 8.0)
    points = centre + r[:, None] * d
    s0 = 1.5 * r[:, None] / fx
    log_scales = torch.log(s0) + 0.5 * torch.randn(n, 3, generator=g)
    return dict(bg_points=points.float(), bg_opacity_logits=torch.logit(torch.rand(n, generator=g) * 0.9 + 0.05),
                bg_log_scales=log_scales.float(), bg_quats=torch.randn(n, 4, generator=g),
                bg_sh_dc=torch.randn(n, 1, 3, generator=g), bg_sh_rest=torch.randn(n, sh_coeffs - 1, 3, generator=g) * 0.1)


def frosting_attributes(params, mesh):
    """Learnable parameters -> rasterizer inputs, as Frosting's properties do (frosting_model.py:713-799)."""
    faces = mesh["faces"].long()
    shell = torch.stack([mesh["inner"], mesh["outer"]], 1)            # n_verts, 2, 3
    cells_verts = shell[faces].transpose(-2, -3)                      # n_faces, 2, 3, 3
    bary = torch.softmax(params["bary_logits"], dim=-1)
    points = (bary[..., None] * cells_verts[mesh["cells"]].reshape(-1, 6, 3)).sum(dim=-2)
    return dict(
        means3D=points,
        opacities=torch.sigmoid(params["opacity_logits"].view(-1, 1)),
        scales=torch.exp(params["log_scales"]),
        rotations=torch.nn.functional.normalize(params["quats"], dim=-1),
        shs=torch.cat([params["sh_dc"], params["sh_rest"]], dim=1),
    )


def frosting_background_attributes(params):
    """Background parameters -> rasterizer inputs, as Frosting's bg_* properties do (frosting_model.py:801-876): points
    as they are, sigmoid, cat(dc, rest), exp, normalize."""
    return dict(
        means3D=params["bg_points"],
        opacities=torch.sigmoid(params["bg_opacity_logits"].view(-1, 1)),
        scales=torch.exp(params["bg_log_scales"]),
        rotations=torch.nn.functional.normalize(params["bg_quats"], dim=-1),
        shs=torch.cat([params["bg_sh_dc"], params["bg_sh_rest"]], dim=1),
    )


# ---- edited / animated scenes (SURVEY.md row a21): the simple adaptation of make_editable, restated ----
# pytorch3d pieces (Meshes normals, matrix_to_quaternion, quaternion_multiply / invert / to_matrix), restated from their
# documented definitions: pytorch3d is not a dependency.  The golden generator (tests/golden/make_frosting_edit_golden.py)
# runs the reference's own source on top of these same restatements, so they are restated, not pinned.

def p3d_faces_normals(verts, faces):
    """Meshes.faces_normals_packed: cross(v1 - v0, v2 - v0) / max(|.|, 1e-6)."""
    fv = verts[faces.long()]
    n = torch.linalg.cross(fv[:, 1] - fv[:, 0], fv[:, 2] - fv[:, 0], dim=-1)
    return n / n.norm(dim=-1, keepdim=True).clamp_min(1e-6)


def p3d_verts_normals(verts, faces):
    """Meshes.verts_normals_packed: the area-weighted face normals cross(v2 - v1, v0 - v1) summed per vertex, normalised
    with eps 1e-6."""
    fl = faces.long()
    fv = verts[fl]
    fn = torch.linalg.cross(fv[:, 2] - fv[:, 1], fv[:, 0] - fv[:, 1], dim=-1)
    n = torch.zeros_like(verts)
    for k in range(3):
        n = n.index_add(0, fl[:, k], fn)
    return torch.nn.functional.normalize(n, eps=1e-6, dim=1)


def standardize_quaternion(q):
    return torch.where(q[..., :1] < 0, -q, q)


def quaternion_multiply(a, b):
    """Hamilton product of (w, x, y, z) quaternions, real part made non-negative."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return standardize_quaternion(torch.stack([
        aw * bw - ax * bx - ay * by - az * bz,
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by - ax * bz + ay * bw + az * bx,
        aw * bz + ax * by - ay * bx + az * bw], -1))


def quaternion_invert(q):
    return q * q.new_tensor([1.0, -1.0, -1.0, -1.0])


def quaternion_to_matrix(q):
    r, i, j, k = q.unbind(-1)
    two_s = 2.0 / (q * q).sum(-1)
    m = torch.stack([1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)], -1)
    return m.reshape(q.shape[:-1] + (3, 3))


def quaternion_apply(q, v):
    """q * (0, v) * quaternion_invert(q), vector part: pytorch3d's quaternion_apply (no normalisation of q, so a
    non-unit q also scales by |q|^2)."""
    p = quaternion_raw_multiply(quaternion_raw_multiply(q, torch.cat([v.new_zeros(v.shape[:-1] + (1,)), v], -1)),
                                quaternion_invert(q))
    return p[..., 1:]


def quaternion_raw_multiply(a, b):
    """Hamilton product of (w, x, y, z) quaternions, without standardisation."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def matrix_to_quaternion(m):
    """The candidate quaternion of the largest |q_c| (first on ties), over 2 max(|q_c|, 0.1); standardised."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.reshape(m.shape[:-2] + (9,)).unbind(-1)
    arg = torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], -1)
    qa = torch.where(arg > 0, arg.clamp_min(0).sqrt(), torch.zeros_like(arg))
    cand = torch.stack([
        torch.stack([qa[..., 0] ** 2, m21 - m12, m02 - m20, m10 - m01], -1),
        torch.stack([m21 - m12, qa[..., 1] ** 2, m10 + m01, m02 + m20], -1),
        torch.stack([m02 - m20, m10 + m01, qa[..., 2] ** 2, m12 + m21], -1),
        torch.stack([m10 - m01, m20 + m02, m21 + m12, qa[..., 3] ** 2], -1)], -2)
    cand = cand / (2.0 * qa[..., None].clamp_min(0.1))
    pick = qa.argmax(-1)
    return standardize_quaternion(torch.gather(cand, -2, pick[..., None, None].expand(pick.shape + (1, 4)))[..., 0, :])


_SH_C0, _SH_C1 = 0.28209479177387814, 0.4886025119029199
_SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
_SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
          1.445305721320277, -0.5900435899266435)


def sh_colors(shs, dirs, deg):
    """RGB of SH rows `shs` [N,M,3] (M >= (deg+1)^2) at unit directions [N,3]: the 3DGS basis, + 0.5, clamp_min 0."""
    x, y, z = (d[:, None] for d in dirs.unbind(-1))
    c = shs
    r = _SH_C0 * c[:, 0]
    if deg > 0:
        r = r - _SH_C1 * y * c[:, 1] + _SH_C1 * z * c[:, 2] - _SH_C1 * x * c[:, 3]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        r = (r + _SH_C2[0] * xy * c[:, 4] + _SH_C2[1] * yz * c[:, 5] + _SH_C2[2] * (2 * zz - xx - yy) * c[:, 6]
             + _SH_C2[3] * xz * c[:, 7] + _SH_C2[4] * (xx - yy) * c[:, 8])
    if deg > 2:
        r = (r + _SH_C3[0] * y * (3 * xx - yy) * c[:, 9] + _SH_C3[1] * xy * z * c[:, 10]
             + _SH_C3[2] * y * (4 * zz - xx - yy) * c[:, 11] + _SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * c[:, 12]
             + _SH_C3[4] * x * (4 * zz - xx - yy) * c[:, 13] + _SH_C3[5] * z * (xx - yy) * c[:, 14]
             + _SH_C3[6] * x * (xx - 3 * yy) * c[:, 15])
    return (r + 0.5).clamp_min(0.0)


def _centroid_dists(verts, fl):
    fv = verts[fl]
    return (fv - fv.mean(dim=-2, keepdim=True)).norm(dim=-1)           # [F,3]


def face_quaternions(verts, faces):
    """compute_face_quaternions: the frame [n, normalize(v0 - v1), normalize(n x R1)] as a unit quaternion."""
    fv = verts[faces.long()]
    nrm = torch.nn.functional.normalize
    r0 = nrm(p3d_faces_normals(verts, faces), dim=-1)
    r1 = nrm(fv[:, 0] - fv[:, 1], dim=-1)
    r2 = nrm(torch.linalg.cross(r0, r1, dim=-1), dim=-1)
    return nrm(matrix_to_quaternion(torch.stack([r0, r1, r2], -1)), dim=-1)


def cell_transformations(verts, faces, edition_mask=None, thickness_rescaling="median", fix_singular=False):
    """compute_cell_transformations(faces_mask=edition_mask) (frosting_model.py:900-967): [F,3,3] transforms from the
    canonical cell to the world, columns [a', b', normalize(n) * d] -- the axis_bary_shifts axes a, b with the shorter
    Gram-Schmidt-orthogonalised against the longer, each in its own slot; d the median of the edited faces' centroid
    distances (median) or the face's own median distance, 0 -> 1 (triangle).  Zero on unedited faces.
    `fix_singular`: make_editable's fix-up where det(T) == 0 (:1073-1112): a zero column 0 becomes c1 x c2, then a zero
    column 1 becomes c2 x c0."""
    fl = faces.long()
    F = fl.shape[0]
    em = torch.ones(F, dtype=torch.bool, device=verts.device) if edition_mask is None else edition_mask.bool()
    fv = verts[fl]
    r2, r6 = math.sqrt(2), math.sqrt(6)
    shifts = torch.tensor([[-r2 / 2, r2 / 2, 0.0], [-1 / r6, -1 / r6, 2 / r6]], dtype=torch.float32, device=verts.device)
    ax = (shifts[None, :, :, None] * fv[:, None]).sum(dim=-2)          # [F,2,3]: v0, v1, v2 terms summed in order
    d_all = _centroid_dists(verts, fl)
    if thickness_rescaling == "median":
        d = d_all[em].median()
    elif thickness_rescaling == "triangle":
        d = torch.ones(F, device=verts.device)
        d[em] = d_all[em].median(dim=-1).values
        d = torch.where(d == 0, torch.ones_like(d), d)[:, None]
    else:
        raise ValueError(f"thickness rescaling method {thickness_rescaling!r} is not recognized")
    n = torch.nn.functional.normalize(p3d_faces_normals(verts, faces), dim=-1) * d
    a, b = ax[:, 0], ax[:, 1]
    swap = (b.norm(dim=-1) > a.norm(dim=-1))[:, None]                   # the longer axis first; a first on ties
    first, second = torch.where(swap, b, a), torch.where(swap, a, b)
    ortho = second - ((second * first).sum(dim=-1, keepdim=True) * first / (first ** 2).sum(dim=-1, keepdim=True))
    T = torch.stack([torch.where(swap, ortho, first), torch.where(swap, first, ortho), n], -1)
    T = torch.where(em[:, None, None], T, torch.zeros_like(T))
    if fix_singular:
        sing = em & (torch.linalg.det(T) == 0)
        if bool(sing.any()):
            t = T[sing]
            z0 = (t[..., 0] == 0).all(dim=-1)
            t[z0, :, 0] = torch.linalg.cross(t[z0, :, 1], t[z0, :, 2], dim=-1)
            z1 = (t[..., 1] == 0).all(dim=-1)
            t[z1, :, 1] = torch.linalg.cross(t[z1, :, 2], t[z1, :, 0], dim=-1)
            T[sing] = t
    return T


def complex_canonical_transforms(params, ref_verts, faces, cells, edition_mask=None, thickness_rescaling="median"):
    """make_editable(use_simple_adapt=False) (frosting_model.py:1055-1119): the canonical transforms
    C = T_ref[cell]^-1 R(normalize(q)) diag(exp(s)) of the edited Gaussians, [P,3,3] with zeros on unedited rows, and
    T_ref.  torch.linalg.solve raises where an edited Gaussian's cell stays singular, as the reference does."""
    F = faces.shape[0]
    em = torch.ones(F, dtype=torch.bool, device=ref_verts.device) if edition_mask is None else edition_mask.bool()
    gem = em[cells]
    T_ref = cell_transformations(ref_verts, faces, em, thickness_rescaling, fix_singular=True)
    G = quaternion_to_matrix(torch.nn.functional.normalize(params["quats"][gem], dim=-1))
    G = G * torch.exp(params["log_scales"][gem])[..., None, :]
    C = torch.zeros((cells.shape[0], 3, 3), dtype=G.dtype, device=G.device)
    C[gem] = torch.linalg.solve(T_ref[cells[gem]], G)
    return C, T_ref


def edited_frosting_attributes(params, ref_verts, faces, cells, inner_dist, outer_dist, verts, campos, sh_degree,
                               edition_mask=None, thickness_rescaling="median", orig_quats=None,
                               deformation_threshold=2.0, adaptation="simple", canonical=None):
    """One frame of an edited Frosting scene in torch, as the reference computes it with make_editable(
    use_simple_adapt=True) (frosting_model.py:649-799, :886-898, :1013-1054; blender/frosting_utils.py:519-571;
    colours :1479-1484 with get_points_rgb :1304-1352).  `ref_verts`: the base vertices make_editable saw; `verts`: this
    frame's.  Returns means3D, opacities, scales, rotations, colors_precomp ([P + n_bg] rows) and the shell (inner,
    outer).  The oracle of frosting_b200.edit.
    `adaptation="complex"`: make_editable(use_simple_adapt=False) -- edited rows from M = T_frame[cell] C
    (get_edited_quaternions_and_scales, :1149-1183): scales the column norms of M (nan_to_num), rotations
    normalize(matrix_to_quaternion(M / max(scales, 1e-10))), a NaN quaternion -> identity.  `canonical`: C [P,3,3] from
    complex_canonical_transforms (computed here when None); the result also carries `cell_T`."""
    fl = faces.long()
    V, F = verts.shape[0], fl.shape[0]
    em = torch.ones(F, dtype=torch.bool, device=verts.device) if edition_mask is None else edition_mask.bool()
    gem = em[cells]
    ref_d, cur_d = _centroid_dists(ref_verts, fl), _centroid_dists(verts, fl)
    if thickness_rescaling == "median":
        # two Python floats (.item()) in the reference: their quotient is formed in double
        f = (cur_d[em].median().double() / ref_d[em].median().double()).float()
        vfac = torch.ones(V, device=verts.device)
        vfac[fl[em].unique()] = f
        gfac = f
    elif thickness_rescaling == "triangle":
        ff = torch.ones(F, device=verts.device)
        ff[em] = (cur_d[em].median(dim=-1).values / ref_d[em].median(dim=-1).values).nan_to_num()
        s = torch.zeros(V, device=verts.device).index_add(0, fl.reshape(-1), ff.repeat_interleave(3))
        cnt = torch.zeros(V, device=verts.device).index_add(0, fl.reshape(-1), torch.ones(3 * F, device=verts.device))
        vfac = s / cnt.clamp(min=1)
        gfac = ff[cells][gem][:, None]
    else:
        raise ValueError(f"thickness rescaling method {thickness_rescaling!r} is not recognized")
    n = p3d_verts_normals(verts, faces)
    inner = verts + vfac[:, None] * inner_dist[:, None] * n
    outer = verts + vfac[:, None] * outer_dist[:, None] * n
    a = frosting_attributes(params, dict(faces=faces, inner=inner, outer=outer, cells=cells))
    c = cells[gem]
    extra = {}
    if adaptation == "simple":
        scales = a["scales"].clone()
        scales[gem] = scales[gem] * gfac
        q = a["rotations"].clone()
        fq, rq = face_quaternions(verts, faces), face_quaternions(ref_verts, faces)
        q[gem] = quaternion_multiply(fq[c], quaternion_multiply(quaternion_invert(rq[c]), q[gem]))
    elif adaptation == "complex":
        if canonical is None:
            canonical, _ = complex_canonical_transforms(params, ref_verts, faces, cells, em, thickness_rescaling)
        T = cell_transformations(verts, faces, em, thickness_rescaling)
        M = T[c] @ canonical[gem]
        s = M.norm(dim=-2)
        scales = a["scales"].clone()
        scales[gem] = s
        scales = scales.nan_to_num()
        q = a["rotations"].clone()
        q[gem] = torch.nn.functional.normalize(matrix_to_quaternion(M / s[..., None, :].clamp_min(1e-10)), dim=-1)
        q[q.isnan().any(dim=-1)] = q.new_tensor([1.0, 0.0, 0.0, 0.0])
        extra = dict(cell_T=T)
    else:
        raise ValueError(f"adaptation {adaptation!r} is not recognized (simple or complex)")
    keep = (cur_d / ref_d).max(dim=-1).values <= deformation_threshold
    opac = a["opacities"].clone()
    opac[gem & ~keep[cells]] = 0.0
    pos, shs = a["means3D"], a["shs"]
    if "bg_points" in params:
        b = frosting_background_attributes(params)
        pos, opac, scales = torch.cat([pos, b["means3D"]]), torch.cat([opac, b["opacities"]]), torch.cat([scales, b["scales"]])
        q, shs = torch.cat([q, b["rotations"]]), torch.cat([shs, b["shs"]])
    dirs = torch.nn.functional.normalize(pos - campos.reshape(1, 3), dim=-1)
    if orig_quats is not None:
        rot = quaternion_to_matrix(quaternion_multiply(q, quaternion_invert(orig_quats)))
        dirs = (dirs[:, None] @ rot)[:, 0]
    colors = sh_colors(shs[:, :(sh_degree + 1) ** 2], dirs, sh_degree)
    return dict(means3D=pos, opacities=opac, scales=scales, rotations=q, colors_precomp=colors, inner=inner, outer=outer,
                **extra)


def deform_base(verts, t=1.0, centre=(0.0, 0.0, 6.0)):
    """A non-rigid deformation of a sphere's base vertices: a twist about y growing with height, a bend, and an
    anisotropic stretch -- so that some faces stretch past ratio 2.  `t` scales it (frames of an animation)."""
    c = verts.new_tensor(centre)
    p = verts - c
    ang = 0.15 * t * p[:, 1]
    ca, sa = torch.cos(ang), torch.sin(ang)
    x = ca * p[:, 0] + sa * p[:, 2]
    z = -sa * p[:, 0] + ca * p[:, 2]
    y = p[:, 1] * (1.0 + 0.8 * t * (p[:, 1] > 1.5).float() * (p[:, 1] - 1.5))
    x = x * (1.0 + 0.35 * t) + 0.08 * t * p[:, 1] ** 2
    z = z * (1.0 - 0.25 * t)
    return torch.stack([x, y, z], -1) + c


# ---- Blender-animated scenes: apply_poses_to_scene (blender/frosting_utils.py:474-516), restated ----
# pytorch3d's Transform3d is restated from its documented maths (a [N,4,4] matrix in the row-vector convention; inverse
# by torch.inverse; transform_points = [p, 1] @ M, then the divide by the homogeneous coordinate); the golden generator
# (tests/golden/make_frosting_skin_golden.py) runs the reference's own source on top of it.

class Transform3d:
    """The slice of pytorch3d.transforms.Transform3d the reference's skinning and SuGaR's depth-normal render use."""

    def __init__(self, dtype=torch.float32, device="cpu", matrix=None):
        self._matrix = torch.eye(4, dtype=dtype, device=device).view(1, 4, 4) if matrix is None else matrix.view(-1, 4, 4)

    def get_matrix(self):
        return self._matrix.clone()

    def inverse(self):
        return Transform3d(matrix=torch.inverse(self._matrix))

    def transform_points(self, points):
        pts = points.clone()
        if pts.dim() == 2:
            pts = pts[None]
        N, P, _ = pts.shape
        pts = torch.cat([pts, torch.ones(N, P, 1, dtype=points.dtype, device=points.device)], dim=2)
        m = self.get_matrix()
        if m.shape[0] != N:
            m = m.expand(N, -1, -1)
        out = pts.bmm(m)
        out = out[..., :3] / out[..., 3:]
        if out.shape[0] == 1 and points.dim() == 2:
            out = out.reshape(points.shape)
        return out

    def transform_normals(self, normals):
        """normals @ inverse(M[:3,:3]^T): the inverse transpose of the linear part, as pytorch3d applies it."""
        mat = self.get_matrix()[:, :3, :3]
        out = (normals if normals.dim() == 3 else normals[None]).bmm(mat.transpose(1, 2).inverse())
        return out.reshape(normals.shape) if normals.dim() == 2 else out


def skin_vertices(package, ref_indices, i_frame, base_verts):
    """apply_poses_to_scene's loop in torch: writes frame `i_frame` (wrapped by the package's frame count) of every rigged
    mesh's range [ref_indices[i], ref_indices[i+1]) of `base_verts` in place and returns it.  `package`: as
    load_blender_package leaves it (float64 weights in `bone_to_vertex_weights`).  The oracle of frosting_b200.skin."""
    n_frames = len(package["camera"]["lens"])
    with torch.no_grad():
        for i_mesh, mesh_dict in enumerate(package["bones"]):
            if not mesh_dict:
                continue
            idx_of, w_of = package["bone_to_vertices"][i_mesh], package["bone_to_vertex_weights"][i_mesh]
            tpose, arm = mesh_dict["vertex"]["tpose_points"], mesh_dict["armature"]
            new_points = torch.zeros_like(tpose)
            for bone, idx in idx_of.items():
                if len(idx) > 0:
                    pose_t = Transform3d(matrix=arm["pose_bones"][bone][i_frame % n_frames].transpose(-1, -2))
                    reset_t = Transform3d(matrix=arm["rest_bones"][bone].transpose(-1, -2)).inverse()
                    new_points[idx] += w_of[bone][..., None] * pose_t.transform_points(
                        reset_t.transform_points(tpose[idx]))
            base_verts[ref_indices[i_mesh]:ref_indices[i_mesh + 1]] = new_points
    return base_verts


def _translation(t):
    m = torch.eye(4, dtype=torch.float64)
    m[:3, 3] = t
    return m


def _rotation(axis, a):
    c, s = math.cos(a), math.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    m = torch.eye(4, dtype=torch.float64)
    m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
    return m


def skinned_rig(verts, n_bones, n_frames, seed=0):
    """A rig over the whole of `verts` (one mesh) as load_blender_package leaves a Blender package -- the keys
    apply_poses_to_scene reads -- and its ref_indices [0, V].  The tracks are the animation's frames.

    The rig is a chain of `n_bones` bones up the y extent of the mesh, T-pose = `verts`.  A vertex at chain coordinate
    u (in bone lengths) takes every bone whose centre lies within h of u, with weight 1 - |u - centre| / h normalised in
    float64; h runs from 0.6 to 2 around the chain, so a vertex has one bone near a bone's centre and up to four in the
    blend zones.  Frame f bends each bone about z and x by angles that vary with the frame and the bone (at most
    0.6 / n_bones and 0.3 / n_bones rad per bone), and moves the root."""
    dev = verts.device
    v = verts.detach().cpu().double()
    lo, hi = v.min(0).values, v.max(0).values
    c = (lo + hi) / 2
    L = float(hi[1] - lo[1]) / n_bones
    u = ((v[:, 1] - lo[1]) / L).clamp(0.0, n_bones - 1e-6)
    h = 0.6 + 0.7 * (1.0 + torch.sin(3.0 * torch.atan2(v[:, 2] - c[2], v[:, 0] - c[0])))
    rows, bones, ws = [], [], []
    for j in range(-2, 3):
        k = u.floor().long() + j
        w = (1.0 - (u - (k.double() + 0.5)).abs() / h).clamp_min(0.0)
        ok = (k >= 0) & (k < n_bones) & (w > 0)
        rows.append(torch.nonzero(ok)[:, 0])
        bones.append(k[ok])
        ws.append(w[ok])
    rows, bones, ws = torch.cat(rows), torch.cat(bones), torch.cat(ws)
    ws = ws / torch.zeros(v.shape[0], dtype=torch.float64).index_add(0, rows, ws)[rows]
    order = torch.argsort(bones * v.shape[0] + rows)
    rows, bones, ws = rows[order], bones[order], ws[order]
    counts = torch.bincount(bones, minlength=n_bones).tolist()
    names = [f"bone_{k:03d}" for k in range(n_bones)]
    heads = [torch.tensor([float(c[0]), float(lo[1]) + k * L, float(c[2])], dtype=torch.float64) for k in range(n_bones)]
    g = torch.Generator().manual_seed(seed)
    phase = torch.rand(n_bones, 2, generator=g, dtype=torch.float64) * 2 * math.pi
    rest, pose = {}, {}
    tracks = torch.empty(n_bones, n_frames, 4, 4, dtype=torch.float64)
    for f in range(n_frames):
        t = 2 * math.pi * f / n_frames
        parent = _translation(heads[0] + torch.tensor([0.1 * math.sin(t), 0.0, 0.05 * math.cos(t)], dtype=torch.float64))
        for k in range(n_bones):
            if k > 0:
                parent = tracks[k - 1, f] @ _translation(heads[k] - heads[k - 1])
            rot = _rotation(2, 0.6 / n_bones * math.sin(t + phase[k, 0].item())) @ \
                _rotation(0, 0.3 / n_bones * math.cos(t + phase[k, 1].item()))
            tracks[k, f] = parent @ rot
    for k, name in enumerate(names):
        rest[name] = _translation(heads[k]).float().to(dev)
        pose[name] = tracks[k].float().to(dev)
    idx_of, w_of = {}, {}
    for name, chunk_r, chunk_w in zip(names, rows.split(counts), ws.split(counts)):
        idx_of[name] = chunk_r.to(dev) if len(chunk_r) else []
        w_of[name] = chunk_w.to(dev) if len(chunk_w) else []
    eye = torch.eye(4, device=dev)
    package = {"camera": {"lens": torch.full((n_frames,), 50.0)},
               "bones": [{"vertex": {"tpose_points": verts.detach().float().contiguous(), "matrix_world": eye},
                          "armature": {"matrix_world": eye, "rest_bones": rest, "pose_bones": pose}}],
               "bone_to_vertices": [idx_of], "bone_to_vertex_weights": [w_of]}
    return package, [0, v.shape[0]]


# ---- texture bake (SURVEY.md row a22): compute_textured_mesh_for_frosting_mesh, restated ----
SH_C0 = 0.28209479177387814          # frosting_utils/spherical_harmonics.py C0; SH2RGB(sh) = sh * C0 + 0.5


def texture_uv_layout(n_faces, square_size, device="cpu"):
    """The UV atlas of texture.py:30-71: (verts_uv [6 n^2, 2] float32, faces_uv [F,3] int64, n, T).  Face f uses UV
    vertices 3f..3f+2 -- half f % 2 of square f // 2, whose cell (i, j) = divmod(f // 2, n) -- with inset corners.
    The division by T is IEEE fp32 on either device, as in the reference run on the CPU and in csrc/texture.cu: T is a
    tensor on `device` (torch's CUDA division by a Python scalar multiplies by its reciprocal instead)."""
    n = int(math.sqrt(n_faces // 2 + 1) + 1)
    T = square_size * n
    ij = torch.cartesian_prod(torch.arange(n, device=device), torch.arange(n, device=device))[:, None]
    u = torch.tensor([[1, 0]], dtype=torch.int32, device=device)[:, None]
    v = torch.tensor([[0, 1]], dtype=torch.int32, device=device)[:, None]
    uv = torch.cat([ij + u, ij, ij + u + v, ij + v, ij, ij + u + v], dim=1) * square_size
    uv = uv + torch.tensor([[-2, 1], [2, 1], [-2, -3], [1, -1], [1, 3], [-3, -1]], device=device)
    verts_uv = uv.reshape(-1, 2).float() / torch.tensor(float(T), device=device)
    faces_uv = torch.arange(3 * n_faces, device=device).view(n_faces, 3)
    return verts_uv, faces_uv, n, T


def _last_wins(idx, n):
    """Positions (into idx) of the last occurrence of every distinct value: the entries that
    `acc[idx] = acc[idx] + x` keeps when idx has duplicates and runs in order, as it does on the CPU."""
    pos = torch.arange(idx.shape[0], device=idx.device)
    win = torch.full((n,), -1, dtype=torch.long, device=idx.device).scatter_reduce_(0, idx, pos, "amax")
    return win[win >= 0]


def bake_texture_torch(n_faces, cells, sh_dc, square_size, images, pix_to_faces, barys):
    """texture.py:11-166 in torch over given views: images [H,W,3] (the render, before nan_to_num / clamp),
    pix_to_faces [H,W] (-1: background) and barys [H,W,3].  Returns (verts_uv, faces_uv, texture [T,T,3]).

    The per-view `acc[idx] = acc[idx] + colors` keeps the last pixel in row-major order of every face and texel
    (_last_wins), as the reference does on the CPU, so the bake is deterministic on either device.  The reference's count
    clamp of the SH colours is an expression whose result is dropped: a face with neither Gaussians nor hits is 0 / 0 =
    NaN, kept here.  Works on CPU and CUDA tensors alike (the CPU run is the oracle of frosting_b200.texture)."""
    device = cells.device
    F = int(n_faces)
    verts_uv, faces_uv, n, T = texture_uv_layout(F, square_size, device)
    uvs = torch.cartesian_prod(torch.arange(T, device=device, dtype=torch.int32),
                               torch.arange(T, device=device, dtype=torch.int32)).view(T, T, 2)
    square = uvs // square_size
    square = square[..., 0] * n + square[..., 1]
    in_top = uvs % square_size
    in_top = in_top[..., 0] < in_top[..., 1]
    uv_to_faces = (2 * square + in_top).transpose(0, 1).clamp_max(F - 1)
    del uvs, square, in_top

    texture_img = torch.zeros(T, T, 3, device=device)
    texture_count = torch.zeros(T, T, 1, device=device)
    face_colors = torch.zeros(F, 3, device=device)
    face_count = torch.zeros(F, 1, device=device)
    cells = cells.long()
    sh_colors = torch.zeros_like(face_colors).index_add_(0, cells, (sh_dc.reshape(-1, 3) * SH_C0 + 0.5).clamp(0., 1.))
    sh_counts = torch.zeros_like(face_count).index_add_(0, cells, torch.ones_like(cells[..., None]).float())
    sh_colors = sh_colors / sh_counts

    for image, p2f, bary in zip(images, pix_to_faces, barys):
        rgb = image.nan_to_num().clamp(min=0, max=1).reshape(-1, 3)
        p2f = p2f.reshape(-1).long()
        mask = p2f > -1
        face_indices, colors = p2f[mask], rgb[mask]
        bary = bary.reshape(-1, 3)[mask]
        w = _last_wins(face_indices, F)
        fw = face_indices[w]
        face_count[fw] = face_count[fw] + 1
        face_colors[fw] = face_colors[fw] + colors[w]
        pix = ((verts_uv[faces_uv[face_indices]] * bary[:, :, None]).sum(dim=1) * T).int()
        ok = ((pix >= 0) & (pix < T)).all(dim=1)
        t = pix[:, 1].long() * T + pix[:, 0].long()
        t = torch.where(ok, t, T * T)                  # outside the texture: a slot past the end, dropped
        w = _last_wins(t, T * T + 1)
        w = w[t[w] < T * T]
        row, col = pix[w, 1].long(), pix[w, 0].long()
        texture_img[row, col] = texture_img[row, col] + colors[w]
        texture_count[row, col] = texture_count[row, col] + 1

    filled = texture_count[..., 0] > 0
    texture_img[filled] = texture_img[filled] / texture_count[filled]
    visited = face_count[..., 0] > 0
    face_colors[visited] = face_colors[visited] / face_count[visited]
    face_colors[~visited] = sh_colors[~visited]
    texture_img[~filled] = face_colors[uv_to_faces[~filled]]
    return verts_uv, faces_uv, texture_img.flip(0)


# ---- SuGaR coarse-stage scenes (SURVEY.md row a23): the SDF regulariser's inputs ----

def sugar_scene(P, seed, K=16, straggler_frac=0.1, device="cpu"):
    """A SuGaR-like coarse scene of P Gaussians as the trainer holds them after activation: flat Gaussians on a bumpy
    sphere (radius 2 around (0, 0, 6), in front of `make_camera`'s default camera), the thin axis along the surface normal
    and at a random index, plus `straggler_frac` volumetric Gaussians scattered around it.  Returns points [P,3],
    scaling [P,3], unit quaternions [P,4], strengths [P,1] and the K-nearest-neighbour table knn_idx [P,K] (int64,
    scipy cKDTree, self first, as pytorch3d knn_points on distinct points)."""
    from scipy.spatial import cKDTree
    g = torch.Generator().manual_seed(seed)
    n_flat = P - int(straggler_frac * P)
    d = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    bump = 1.0 + 0.08 * torch.sin(5 * d[:, 0]) * torch.cos(4 * d[:, 1])
    spacing = math.sqrt(4 * math.pi * 4.0 / max(P, 1))
    centre = torch.tensor([0.0, 0.0, 6.0])
    points = centre + 2.0 * bump[:, None] * d
    scaling = spacing * torch.exp(0.3 * torch.randn(P, 3, generator=g))
    # the normal axis: a random column of a random frame whose column c is the sphere's normal
    c = torch.randint(0, 3, (P,), generator=g)
    t1 = torch.nn.functional.normalize(torch.linalg.cross(d, torch.randn(P, 3, generator=g), dim=-1), dim=-1)
    t2 = torch.linalg.cross(d, t1, dim=-1)
    R = torch.zeros(P, 3, 3)
    for k in range(3):
        pick = c == k
        R[pick, :, k] = d[pick]
        R[pick, :, (k + 1) % 3] = t1[pick]
        R[pick, :, (k + 2) % 3] = t2[pick]
    thin = spacing * 0.02 * torch.exp(0.5 * torch.randn(P, generator=g))
    scaling[torch.arange(P), c] = thin
    q = matrix_to_quaternion(R)
    # stragglers: volumetric, anywhere within 0.3 of the surface, random orientation
    s = slice(n_flat, P)
    points[s] += 0.3 * torch.randn(P - n_flat, 3, generator=g)
    scaling[s] = 3 * spacing * torch.exp(0.3 * torch.randn(P - n_flat, 3, generator=g))
    q[s] = torch.randn(P - n_flat, 4, generator=g)
    q = torch.nn.functional.normalize(q, dim=-1)
    strengths = torch.sigmoid(2.0 * torch.randn(P, 1, generator=g))
    knn = torch.from_numpy(cKDTree(points.double().numpy()).query(points.double().numpy(), k=K)[1]).long().reshape(P, K)
    to =lambda t: t.contiguous().to(device)
    return dict(points=to(points), scaling=to(scaling), quaternions=to(q), strengths=to(strengths), knn_idx=to(knn))


# ---- point sets for the exact K-nearest-neighbour search (knn.py) ----

KNN_SCENES = ("sugar", "cube", "plane", "line", "lattice", "coincident", "offset")


def knn_scene(kind, P, seed, outlier_frac=0.01):
    """float32 [P,3] point sets (CPU) for knn_points:
      sugar       a SuGaR-like coarse scene: centres on the bumpy sphere of `sugar_scene`, 10 % scattered within 0.3
                  of it, and `outlier_frac` far background Gaussians at 10 to 10^4 surface spacings beyond it
      cube        uniform in the unit cube
      plane       uniform in a square, z constant
      line        uniform on a segment
      lattice     the integer lattice n^3 (P = n^3), in a random order: most distances tie exactly
      coincident  min(5000, P // 2) copies of one point, the rest pairs of clones, in a random order
      offset      a small sphere near (1000, 1000, 1000) with spacing ~1e-3: distances near the float32 rounding
    """
    g = torch.Generator().manual_seed(seed)
    if kind == "sugar":
        d = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
        bump = 1.0 + 0.08 * torch.sin(5 * d[:, 0]) * torch.cos(4 * d[:, 1])
        pts = torch.tensor([0.0, 0.0, 6.0]) + 2.0 * bump[:, None] * d
        spacing = math.sqrt(4 * math.pi * 4.0 / max(P, 1))
        n_far = int(outlier_frac * P)
        n_near = int(0.1 * P)
        pts[P - n_near - n_far:P - n_far] += 0.3 * torch.randn(n_near, 3, generator=g)
        far = torch.nn.functional.normalize(torch.randn(n_far, 3, generator=g), dim=-1)
        dist = 2.0 + spacing * 10.0 ** (1 + 3 * torch.rand(n_far, 1, generator=g))
        pts[P - n_far:] = torch.tensor([0.0, 0.0, 6.0]) + dist * far
        return pts[torch.randperm(P, generator=g)].contiguous()
    if kind == "cube":
        return torch.rand(P, 3, generator=g)
    if kind == "plane":
        pts = torch.rand(P, 3, generator=g)
        pts[:, 2] = 0.25
        return pts
    if kind == "line":
        t = torch.rand(P, 1, generator=g)
        return (torch.tensor([0.1, -0.2, 3.0]) + t * torch.tensor([1.0, 0.5, -0.25])).contiguous()
    if kind == "lattice":
        n = round(P ** (1 / 3))
        if n ** 3 != P:
            raise ValueError(f"a lattice needs a cube P, got {P}")
        a = torch.arange(n, dtype=torch.float32)
        pts = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(P, 3)
        return pts[torch.randperm(P, generator=g)].contiguous()
    if kind == "coincident":
        m = min(5000, P // 2)
        pairs = torch.rand((P - m + 1) // 2, 3, generator=g).repeat_interleave(2, 0)[:P - m]
        pts = torch.cat([torch.full((m, 3), 0.5), pairs])
        return pts[torch.randperm(P, generator=g)].contiguous()
    if kind == "offset":
        r = 1e-3 * math.sqrt(P / (4 * math.pi))
        d = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
        return (torch.tensor([1000.0, 1000.0, 1000.0]) + r * d).contiguous()
    raise ValueError(f"unknown knn scene {kind!r}; one of {KNN_SCENES}")
