"""Golden vectors for SuGaR's depth-normal consistency, produced by EXECUTING the reference's own source.

From frosting_scene/sugar_model.py, the methods `get_smallest_axis`, `get_normals` and `render_depth_and_normal` are cut
out of class SuGaR with `ast` and bound to a stub model holding the activated tensors (points, scaling, quaternions).
Its `render_image_gaussian_rasterizer` is a stub that records the `point_colors` it receives (the features) and returns
a given image `dn` [3,H,W] channels-last, as the rasterizer's output is.  From
frosting_trainers/coarse_density_and_dn_consistency.py, `depths_to_points`, `depth2normal_2dgs` and
`depth_normal_consistency_loss` are cut out the same way.  The trainer's call (:649-656) is then made: features, the
normal image of `dn`, and the loss with scale_rendered_normals=False.

The pytorch3d camera is stood in by frosting_b200.scenes.Transform3d with R and T built as
frosting_scene/cameras.py:276-322 builds them from the GSCamera (R = W2C[:3,:3]^T, T = W2C[:3,3]), in the run's dtype;
get_camera_center is pytorch3d's (the inverse world-to-view matrix's translation row).  The GSCamera is
frosting_b200.scenes.make_camera's (world_view_transform, full_proj_transform, image size).

Textual substitutions in the cut source, each touching only device or dtype (DTYPE is the run's dtype):
  `.float().cuda()`       -> `.to(DTYPE)`          (ndc2pix in depths_to_points)
  `device='cuda'`         -> `device='cpu'`        (the pixel grid)
  `.float()`              -> `.to(DTYPE)`          (the pixel grid; render_depth_and_normal's bg_color)

Run under torch.use_deterministic_algorithms(True).  Inputs are float32; each is evaluated in float64 (the float32
inputs cast) and in float32.  Stored per precision: the features and their gradients with respect to points, scaling and
quaternions for a seeded cotangent; per image case the loss and dL/ddn.

Features: 300 Gaussians of frosting_b200.scenes.sugar_scene plus tied scales (two and three equal axes) and a normal
perpendicular to the view ray (sign 0, exact in float32), under a camera whose rotation is a cyclic permutation (exact
arithmetic in the stand-in's inverses).  Images: 1x1, 2x5, 3x3, 23x37 (odd, not square) and 40x64 under a rotated
look-at camera, and 23x37 under the permutation camera; depth is a smooth surface with a background region of depth
0 and a step discontinuity, normal channels have pixels with |xy|^2 > 1.

    python tests/golden/make_sugar_dn_golden.py        # writes tests/golden/loss_sugar_dn.npz

The checkout is found as oracle/build_ref.py finds it ($FROSTING_REFERENCE, else `reference/` beside the repository).
"""
import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_dir      # noqa: E402
from frosting_b200 import scenes                # noqa: E402

P, SEED = 300, 20261018
METHODS = ("get_smallest_axis", "get_normals", "render_depth_and_normal")
FUNCTIONS = ("depths_to_points", "depth2normal_2dgs", "depth_normal_consistency_loss")
SUBSTITUTIONS = ((".float().cuda()", ".to(DTYPE)"), ("device='cuda'", "device='cpu'"), (".float()", ".to(DTYPE)"))
# (name, H, W, camera)
IMAGES = (("1x1", 1, 1, "look"), ("2x5", 2, 5, "look"), ("3x3", 3, 3, "look"), ("23x37", 23, 37, "look"),
          ("40x64", 40, 64, "look"), ("23x37_perm", 23, 37, "perm"))


def _cut(path, names, cls=None):
    src = open(path).read()
    lines = src.splitlines()
    body = ast.parse(src).body
    if cls is not None:
        body = next(n for n in body if isinstance(n, ast.ClassDef) and n.name == cls).body
    out = [textwrap.dedent("\n".join(lines[n.lineno - 1:n.end_lineno])) for n in body
           if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(out) == len(names), path
    text = "\n\n".join(out) + "\n"
    for a, b in SUBSTITUTIONS:
        text = text.replace(a, b)
    return text


def cameras():
    """W2C of the two cameras: a cyclic permutation with an integer translation, and a rotated look-at camera."""
    perm = torch.eye(4)
    perm[:3, :3] = torch.tensor([[0.0, 1.0, 0.0], [0.0, 0.0, 1.0], [1.0, 0.0, 0.0]])
    perm[:3, 3] = torch.tensor([1.0, -2.0, 3.0])
    return {"perm": perm, "look": scenes.look_at_w2c((1.5, -0.7, 0.4), (0.0, 0.2, 6.0))}


def make_gaussians():
    sc = scenes.sugar_scene(P, 5, K=1)
    pts, scl, q = sc["points"], sc["scaling"], sc["quaternions"]
    scl[3] = torch.tensor([0.02, 0.02, 0.05])         # tied: the first of two minimal axes
    scl[4] = torch.tensor([0.03, 0.03, 0.03])         # all three tied
    scl[5] = torch.tensor([0.05, 0.01, 0.01])
    # normal e_x (identity quaternion, smallest axis 0), camera centre - p along e_y: n . (c - p) == 0 exactly
    w2c = cameras()["perm"]
    centre = -(w2c[:3, :3].T @ w2c[:3, 3])
    q[6] = torch.tensor([1.0, 0.0, 0.0, 0.0])
    scl[6] = torch.tensor([0.001, 0.02, 0.03])
    pts[6] = centre + torch.tensor([0.0, 4.0, 0.0])
    q[7] = q[7] * 1.7                                  # raw, not unit: two_s = 2 / |q|^2
    g = torch.Generator().manual_seed(SEED)
    cot = torch.randn(P, 3, generator=g)
    return dict(points=pts, scaling=scl, quaternions=q, cot=cot)


def make_image(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    depth = 5.0 + 0.4 * torch.sin(0.3 * x) * torch.cos(0.2 * y) + 0.01 * x
    depth = torch.where(x > 0.6 * W, depth + 1.0, depth)                      # step discontinuity
    depth = torch.where((y < 0.3 * H) & (x < 0.3 * W), torch.zeros_like(depth), depth)   # background
    nxy = 0.6 * (2 * torch.rand(2, H, W, generator=g, dtype=torch.float64) - 1)
    over = torch.rand(H, W, generator=g, dtype=torch.float64) < 0.1
    nxy[:, over] = torch.tensor([0.9, -0.8], dtype=torch.float64)[:, None]   # |xy|^2 = 1.45 > 1
    return torch.cat([depth[None], nxy]).float().contiguous()


def p3d_camera(w2c32, dtype):
    """R, T as frosting_scene/cameras.py:276-322 makes them from the GSCamera's R = W2C[:3,:3]^T, T = W2C[:3,3]."""
    R = w2c32[:3, :3].T.to(dtype)[None]
    T = w2c32[:3, 3].to(dtype)[None]
    w2c = torch.zeros(1, 4, 4, dtype=dtype)
    w2c[:, :3, :3] = R.transpose(-1, -2)
    w2c[:, :3, 3] = T
    w2c[:, 3, 3] = 1
    c2w = w2c.inverse()
    c2w[:, :3, 1:3] *= -1
    c2w = c2w[:, :3, :]
    line = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=dtype).expand(1, -1, -1)
    world2cam = torch.cat([c2w, line], dim=1).inverse()
    R, T = world2cam.split([3, 1], dim=-1)
    R = R[:, :3].transpose(1, 2) * torch.tensor([-1.0, 1.0, -1], dtype=dtype)
    T = T.squeeze(2)[:, :3] * torch.tensor([-1.0, 1.0, -1], dtype=dtype)
    M = torch.zeros(1, 4, 4, dtype=dtype)
    M[:, :3, :3] = R
    M[:, 3, :3] = T
    M[:, 3, 3] = 1
    w2v = scenes.Transform3d(matrix=M)
    return types.SimpleNamespace(get_world_to_view_transform=lambda: w2v,
                                 get_camera_center=lambda: w2v.inverse().get_matrix()[:, 3, :3])


def main():
    torch.use_deterministic_algorithms(True)
    root = reference_dir()
    model_py = os.path.join(root, "frosting_scene", "sugar_model.py")
    trainer_py = os.path.join(root, "frosting_trainers", "coarse_density_and_dn_consistency.py")
    if not os.path.exists(model_py):
        raise SystemExit(f"{model_py} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
    methods, functions = _cut(model_py, METHODS, cls="SuGaR"), _cut(trainer_py, FUNCTIONS)

    gs = make_gaussians()
    w2cs = cameras()
    images = {name: make_image(H, W, i) for i, (name, H, W, _) in enumerate(IMAGES)}
    save = {k: v.numpy() for k, v in gs.items()}
    for name, w2c in w2cs.items():
        cam = scenes.make_camera(64, 40, w2c)
        save[f"cam_{name}/w2c"] = w2c.numpy()
        save[f"cam_{name}/campos"] = cam.camera_center.numpy()
    for name, H, W, camname in IMAGES:
        cam = scenes.make_camera(W, H, w2cs[camname])
        save[f"img_{name}/dn"] = images[name].numpy()
        save[f"img_{name}/view"] = cam.world_view_transform.numpy()
        save[f"img_{name}/proj"] = cam.full_proj_transform.numpy()

    for tag, dtype in (("f32", torch.float32), ("f64", torch.float64)):
        ns = {"torch": torch, "np": np, "quaternion_to_matrix": scenes.quaternion_to_matrix, "DTYPE": dtype}
        exec(compile(methods, model_py, "exec"), ns)
        exec(compile(functions, trainer_py, "exec"), ns)

        def run(camname, H, W, dn, leaves):
            w2c = w2cs[camname]
            gcam = scenes.make_camera(W, H, w2c)
            p3d = p3d_camera(w2c, dtype)
            recorded = {}

            def rasterize(sh_deg, camera_indices, point_colors, bg_color):
                recorded["features"] = point_colors
                return dn.transpose(0, 1).transpose(1, 2)

            model = types.SimpleNamespace(
                points=leaves["points"], scaling=leaves["scaling"], quaternions=leaves["quaternions"], device="cpu",
                binded_to_surface_mesh=False, render_image_gaussian_rasterizer=rasterize,
                nerfmodel=types.SimpleNamespace(training_cameras=types.SimpleNamespace(p3d_cameras=[p3d])))
            for m in METHODS:
                setattr(model, m, types.MethodType(ns[m], model))
            depth_img, normal_img = model.render_depth_and_normal(camera_indices=0)
            gs_camera = types.SimpleNamespace(world_view_transform=gcam.world_view_transform.to(dtype),
                                              full_proj_transform=gcam.full_proj_transform.to(dtype),
                                              image_width=W, image_height=H)
            loss = ns["depth_normal_consistency_loss"](depth=depth_img[None], normal=normal_img.permute(2, 0, 1),
                                                       camera=gs_camera, scale_rendered_normals=False,
                                                       return_normal_maps=False)
            return recorded["features"], loss

        leaves = {k: gs[k].to(dtype).requires_grad_(True) for k in ("points", "scaling", "quaternions")}
        dn = images["3x3"].to(dtype).requires_grad_(True)
        feats, _ = run("perm", 3, 3, dn, leaves)
        save[f"{tag}/features"] = feats.detach().numpy()
        grads = torch.autograd.grad(feats, list(leaves.values()), grad_outputs=gs["cot"].to(dtype), allow_unused=True)
        for k, g in zip(leaves, grads):
            save[f"{tag}/dfeatures_d{k}"] = (torch.zeros_like(leaves[k]) if g is None else g).numpy()
        for name, H, W, camname in IMAGES:
            dn = images[name].to(dtype).requires_grad_(True)
            _, loss = run(camname, H, W, dn, {k: v.detach() for k, v in leaves.items()})
            (g,) = torch.autograd.grad(loss, [dn], allow_unused=True)
            save[f"{tag}/loss_{name}"] = np.array(loss.item())
            save[f"{tag}/dloss_ddn_{name}"] = (torch.zeros_like(dn) if g is None else g).numpy()
    np.savez_compressed(os.path.join(HERE, "loss_sugar_dn.npz"), **save)
    print(len(save), "arrays", sum(v.nbytes for v in save.values()), "bytes; losses f64",
          [float(save[f"f64/loss_{n}"]) for n, *_ in IMAGES])


if __name__ == "__main__":
    main()
