"""Float64 model of the per-Gaussian backward (frosting_b200/csrc/geom_bwd.cu), row by row.

TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

The per-Gaussian backward is linear in the blend backward's 12-float accumulator record of each Gaussian
(fb200_layout.geom_acc): slots 0-8 are the cotangents of the splat's screen-space quantities,
  {dmean2D.x, dmean2D.y, dconic.x, dconic.y}, {dconic.w, dopacity, dr, dg}, {db, -, -, -}.
So every gradient element the kernel writes is  g_i = sum_k J_ik acc_k  with J the Jacobian of the per-Gaussian forward
map below.  That map is written here from the maths in torch float64 and differentiated by autograd; the reference's
backward departs from the exact derivative in four places, and each departure is expressed at the autograd level:
  * scale modifier:   s_eff = s + (mod - 1) s.detach()      value mod * s, d(scale) without the factor mod;
  * quaternion:       R is built from the raw q             (no normalisation, as the forward does);
  * guard band:       outside |t.x / t.z| <= 1.3 tanfov the clamped t.x = clamp(t.x / t.z) t.z enters J as a
                      constant -- no d/dt.x, and d/dt.z holds t.x fixed (the reference's dL/dtz treats the clamped t.x
                      as independent of t.z);
  * conic:            the inverse's derivative is scaled by det^2 / (det^2 + 1e-7);
and the colour clamp uses the forward's own `clamped` bits (fb200_layout.geom_clamped), not a float64 re-decision.
dconic.y is accumulated as half the derivative w.r.t. conic.y (the blend's power has conic.y d.x d.y once): the model's
second conic output is 2 conic.y.

`vjp_by_slot` returns, per gradient element, g64 = sum_k J_ik acc_k and the magnitude m64 = sum_k |J_ik acc_k| (one VJP
per slot, all rows at once).  A float32 evaluation of the same map is within a few ulp of m64 unless a slot's own
contribution cancels internally, so |g32 - g64| <= tau * m64 is a per-element bound with no fraction allowance.
"""
import torch

from frosting_b200 import scenes

# real spherical harmonics up to degree 3 (the constants of the 3DGS colour model)
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)
N_SLOTS = 9          # accumulator slots the per-Gaussian backward reads
GUARD = 1.3          # the guard band: 1.3 tanfov


class Camera:
    """The per-call camera of fb200_params / fb200_inputs in float64.  `view`, `proj`: the 4x4 matrices as stored by
    torch (row vector convention: [p, 1] @ view)."""

    def __init__(self, rs, device=None):
        f32 = lambda v: float(torch.tensor(float(v), dtype=torch.float32))
        device = device or rs.viewmatrix.device
        self.W, self.H = int(rs.image_width), int(rs.image_height)
        self.tanx, self.tany = f32(rs.tanfovx), f32(rs.tanfovy)
        self.fx, self.fy = self.W / (2.0 * self.tanx), self.H / (2.0 * self.tany)
        self.limx, self.limy = GUARD * self.tanx, GUARD * self.tany
        self.view = rs.viewmatrix.detach().to(device, torch.float64).reshape(4, 4)
        self.proj = rs.projmatrix.detach().to(device, torch.float64).reshape(4, 4)
        self.campos = rs.campos.detach().to(device, torch.float64).reshape(3)
        self.mod = f32(rs.scale_modifier)


def sh_basis(d, D):
    """[N, (D+1)^2] basis values at unit directions d [N,3]."""
    x, y, z = d.unbind(-1)
    b = [torch.full_like(x, SH_C0)]
    if D > 0:
        b += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if D > 1:
        xx, yy, zz = x * x, y * y, z * z
        b += [SH_C2[0] * x * y, SH_C2[1] * y * z, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * x * z, SH_C2[4] * (xx - yy)]
    if D > 2:
        b += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * x * y * z, SH_C3[2] * y * (4 * zz - xx - yy),
              SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
              SH_C3[6] * x * (xx - 3 * yy)]
    return torch.stack(b, -1)


def rotation_rows(q):
    """R with Sigma = R^T diag(s)^2 R, from q = (r, x, y, z) as given (not normalised)."""
    r, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], -1),
        torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], -1),
        torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def sym3(c):
    """[N,6] upper triangle (c0 c1 c2; c3 c4; c5) -> [N,3,3]: an off-diagonal parameter enters twice."""
    return torch.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], -2)


def guard_ratio(cam, means):
    """|t.x / t.z| / (1.3 tanfovx), |t.y / t.z| / (1.3 tanfovy) per row, in float64: > 1 outside the guard band."""
    t = torch.cat([means.detach().double(), torch.ones_like(means[:, :1], dtype=torch.float64)], 1) @ cam.view
    return (t[:, 0] / t[:, 2]).abs() / cam.limx, (t[:, 1] / t[:, 2]).abs() / cam.limy


def _guarded(t, tz, lim):
    r = t / tz
    return torch.where(r.abs() <= lim, t, (r.clamp(-lim, lim) * tz).detach())


def projected_cov(cam, means, scales=None, rotations=None, cov3D=None):
    """J W Sigma W^T J^T [N,2,2], before the 0.3 dilation."""
    hom = torch.cat([means, torch.ones_like(means[:, :1])], 1)
    t = hom @ cam.view
    tz = t[:, 2]
    tx, ty = _guarded(t[:, 0], tz, cam.limx), _guarded(t[:, 1], tz, cam.limy)
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([cam.fx / tz, zero, -cam.fx * tx / (tz * tz)], -1),
                     torch.stack([zero, cam.fy / tz, -cam.fy * ty / (tz * tz)], -1)], -2)
    T = J @ cam.view[:3, :3].t()
    if cov3D is not None:
        Sigma = sym3(cov3D)
    else:
        s = scales + (cam.mod - 1.0) * scales.detach()
        R = rotation_rows(rotations)
        Sigma = R.transpose(-1, -2) @ (R * (s * s)[:, :, None])
    return T @ Sigma @ T.transpose(-1, -2)


def splat_map(cam, means, opacity, *, scales=None, rotations=None, cov3D=None, shs=None, colors=None, D=0,
              clamped=None):
    """The per-Gaussian forward map, [N, N_SLOTS] outputs in the accumulator's slot order:
    NDC mean (2), conic (c, -2b, a) / det of cov2D = [[a, b], [b, c]] (3), opacity (1), colour (3).
    Exactly one of (scales + rotations | cov3D) and of (shs | colors); `clamped` [N,3] bool: the forward's colour clamp."""
    N = means.shape[0]
    h = torch.cat([means, torch.ones_like(means[:, :1])], 1) @ cam.proj
    ndc = h[:, :2] / (h[:, 3:4] + 1e-7)
    cov = projected_cov(cam, means, scales, rotations, cov3D)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * c - b * b
    conic = torch.stack([c, -2 * b, a], -1) / det[:, None]
    k = (det * det / (det * det + 1e-7)).detach()
    conic = conic.detach() + (conic - conic.detach()) * k[:, None]
    if shs is not None:
        d = means - cam.campos
        d = d / d.norm(dim=-1, keepdim=True)
        basis = sh_basis(d, D)
        raw = torch.einsum("nk,nkc->nc", basis, shs[:, :basis.shape[1]]) + 0.5
        color = torch.where(clamped, torch.zeros_like(raw), raw)
    else:
        color = colors
    return torch.cat([ndc, conic, opacity.reshape(N, 1), color], 1)


def vjp_by_slot(out, leaves, acc):
    """g64, m64 (dicts shaped like `leaves`) of the outputs `out` [N, N_SLOTS] with cotangent acc[:, :N_SLOTS].

    Every leaf holds one row per output row (its first dimension is N or a multiple of N, rows contiguous), and the rows
    are independent.  m64 is the componentwise condition of g64 w.r.t. everything the kernel reads as float32:
      sum_k |J_ik acc_k|   (one VJP per slot)   +   sum_j |dg_i/dx_j| |x_j|   (one double-backward per column of g),
    the first-order change of g_i when every input moves by its own relative rounding.  The second sum covers the
    cancellations inside J (a basis value 2z^2 - x^2 - y^2 near zero, the terms of d(scale) cancelling, ...) that the
    first cannot see."""
    names = list(leaves)
    xs = [leaves[k] for k in names]
    N = out.shape[0]
    g = {k: torch.zeros_like(leaves[k]) for k in names}
    m = {k: torch.zeros_like(leaves[k]) for k in names}
    acc = acc.to(out)
    for s in range(N_SLOTS):
        cot = torch.zeros_like(out)
        cot[:, s] = acc[:, s]
        gr = torch.autograd.grad(out, xs, cot, retain_graph=True, allow_unused=True)
        for k, v in zip(names, gr):
            if v is not None:
                g[k] += v
                m[k] += v.abs()
    cot = torch.zeros_like(out)
    cot[:, :N_SLOTS] = acc[:, :N_SLOTS]
    gg = torch.autograd.grad(out, xs, cot, create_graph=True, allow_unused=True)
    for k, v in zip(names, gg):
        if v is None or not v.requires_grad:
            continue
        cols = v.reshape(N, -1)
        mk = m[k].view(N, -1)
        for i in range(cols.shape[1]):
            if not bool((cols[:, i] != 0).any()):
                continue
            d = torch.autograd.grad(cols[:, i].sum(), xs, retain_graph=True, allow_unused=True)
            mk[:, i] += sum((dj * xj.detach()).abs().reshape(N, -1).sum(1) for dj, xj in zip(d, xs) if dj is not None)
    return g, m


def _leaf(t):
    return t.detach().to(torch.float64).clone().requires_grad_(True)


def splat_grads(cam, acc, clamped=None, D=0, **inputs):
    """The per-Gaussian backward of plain rasterizer inputs (means3D, opacities and one of each pair of splat_map) for
    the rows given.  Returns g64, m64 by input name."""
    leaves = {k: _leaf(v) for k, v in inputs.items() if v is not None}
    kw = {k: v for k, v in leaves.items() if k not in ("means3D", "opacities")}
    with torch.enable_grad():
        out = splat_map(cam, leaves["means3D"], leaves["opacities"], D=D, clamped=clamped, **kw)
        return vjp_by_slot(out, leaves, acc)


def frosting_grads(cam, acc, clamped, D, params, mesh, mesh_rows, bg_rows):
    """The per-Gaussian backward of frosting mode: gradients of Frosting's parameters for the mesh rows `mesh_rows` and
    the background rows `bg_rows` (indices into the bg_* tensors) of a frame; `acc`, `clamped` are the frame's rows
    (mesh rows first).  The attribute maps are scenes.frosting_attributes / frosting_background_attributes in float64.
    Returns g64, m64: the six mesh parameters and bg_* by name, rows in the order given, and `inner` / `outer` [V,3]
    (scatter-added; m64 scatter-adds the absolute per-row contributions)."""
    dev = acc.device
    g, m = {}, {}
    n_mesh = params["bary_logits"].shape[0]
    with torch.enable_grad():
        if mesh_rows.numel():
            p = {k: _leaf(params[k][mesh_rows]) for k in ("bary_logits", "opacity_logits", "log_scales", "quats",
                                                          "sh_dc", "sh_rest")}
            vid = mesh["faces"].long()[mesh["cells"][mesh_rows]]                       # [n,3]
            n = vid.shape[0]
            corner = {k: _leaf(mesh[k][vid.reshape(-1)]) for k in ("inner", "outer")}  # one copy per row and corner
            rows = dict(faces=torch.arange(3 * n, device=dev).view(n, 3), cells=torch.arange(n, device=dev), **corner)
            a = scenes.frosting_attributes(p, rows)
            out = splat_map(cam, a["means3D"], a["opacities"], scales=a["scales"], rotations=a["rotations"],
                            shs=a["shs"], D=D, clamped=clamped[mesh_rows])
            gm, mm = vjp_by_slot(out, dict(p, **corner), acc[mesh_rows])
            for k in ("inner", "outer"):
                V = mesh[k].shape[0]
                idx = vid.reshape(-1, 1).expand(-1, 3)
                g[k] = torch.zeros(V, 3, dtype=torch.float64, device=dev).scatter_add_(0, idx, gm.pop(k))
                m[k] = torch.zeros(V, 3, dtype=torch.float64, device=dev).scatter_add_(0, idx, mm.pop(k))
            g.update(gm)
            m.update(mm)
        if bg_rows.numel():
            p = {k: _leaf(params[k][bg_rows]) for k in ("bg_points", "bg_opacity_logits", "bg_log_scales", "bg_quats",
                                                        "bg_sh_dc", "bg_sh_rest")}
            a = scenes.frosting_background_attributes(p)
            fr = bg_rows + n_mesh
            out = splat_map(cam, a["means3D"], a["opacities"], scales=a["scales"], rotations=a["rotations"],
                            shs=a["shs"], D=D, clamped=clamped[fr])
            gb, mb = vjp_by_slot(out, p, acc[fr])
            g.update(gb)
            m.update(mb)
    return g, m


def excess(g32, g64, m64):
    """|g32 - g64| / m64 per element (0 where both sides are exactly 0)."""
    d = (g32.double() - g64).abs()
    return torch.where(d == 0, torch.zeros_like(d), d / m64.clamp_min(1e-300))


def outside(g32, g64, m64, tau):
    """Elements outside the bound |g32 - g64| <= tau m64 + 1e-30, as a boolean mask."""
    return (g32.double() - g64).abs() > tau * m64 + 1e-30
