"""Golden vectors for the texture bake of a Frosting model, produced by EXECUTING the reference's own source.

`compute_textured_mesh_for_frosting_mesh` is cut out of the reference's frosting_utils/texture.py with `ast` (and
`SH2RGB` with its `C0` out of frosting_utils/spherical_harmonics.py) and run unmodified on the CPU.  Stubs stand in for
what it calls:
  - the model's render returns fixed per-view images [H,W,3] (values out of [0, 1], NaN and +-inf included);
  - `MeshRasterizer` returns fixed fragments (pix_to_face, barycentrics with the third weight 1 - (u + v));
  - `Meshes` and `TexturesUV` only hold their arguments.
The inputs: an irregular 37-face mesh (odd: the last square is half used), 50 Gaussians, 3 views of 20x28 pixels where
blocks of pixels share a face and, at these square sizes, a texel.  Faces 3 and 30 are seen by no view, faces 5 and 20
have no Gaussian, faces 12 and 36 neither (their colour is the reference's 0 / 0).  Baked at square_size 3 and 8.

    python tests/golden/make_texture_golden.py        # writes tests/golden/frosting_texture_bake.npz

The checkout is found as oracle/build_ref.py finds it ($FROSTING_REFERENCE, else `reference/` beside the repository).
"""
import ast
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_dir      # noqa: E402

F, V, P, H, W, N_VIEWS = 37, 30, 50, 20, 28, 3
UNSEEN, NO_GAUSSIANS = (3, 12, 30, 36), (5, 12, 20, 36)
SQUARE_SIZES = (3, 8)


def _cut(path, names):
    src = open(path).read()
    lines = src.splitlines()
    out = []
    for n in ast.parse(src).body:
        if (isinstance(n, ast.FunctionDef) and n.name in names) or \
                (isinstance(n, ast.Assign) and any(getattr(t, "id", None) in names for t in n.targets)):
            out.append("\n".join(lines[n.lineno - 1:n.end_lineno]))
    assert len(out) == len(names), (path, names)
    return "\n\n".join(out) + "\n"


class _Meshes:
    def __init__(self, verts, faces, textures=None):
        self.verts, self.faces, self.textures = verts, faces, textures

    def faces_packed(self):
        return self.faces[0]

    def verts_list(self):
        return self.verts

    def faces_list(self):
        return self.faces


class _TexturesUV:
    def __init__(self, maps, verts_uvs, faces_uvs, sampling_mode):
        self.maps, self.verts_uvs, self.faces_uvs, self.sampling_mode = maps, verts_uvs, faces_uvs, sampling_mode


class _Cameras:
    def __init__(self, gs_cameras):
        self.gs_cameras = gs_cameras

    def __len__(self):
        return len(self.gs_cameras)


class _RasterizationSettings:
    def __init__(self, image_size):
        self.image_size = image_size


def reference_namespace(fragments):
    root = reference_dir()
    tex = os.path.join(root, "frosting_utils", "texture.py")
    sh = os.path.join(root, "frosting_utils", "spherical_harmonics.py")
    if not os.path.exists(tex):
        raise SystemExit(f"{tex} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")

    class _MeshRasterizer:
        def __init__(self, cameras, raster_settings, use_nvdiffrast):
            self.cameras = cameras

        def __call__(self, mesh, cam_idx):
            p2f, bary = fragments[cam_idx]
            return SimpleNamespace(pix_to_face=p2f.view(1, H, W, 1), bary_coords=bary.view(1, H, W, 1, 3))

    ns = {"torch": torch, "np": np, "Frosting": object, "Meshes": _Meshes, "TexturesUV": _TexturesUV,
          "MeshRasterizer": _MeshRasterizer, "RasterizationSettings": _RasterizationSettings}
    exec(compile(_cut(sh, ("C0", "SH2RGB")), sh, "exec"), ns)
    exec(compile(_cut(tex, ("compute_textured_mesh_for_frosting_mesh",)), tex, "exec"), ns)
    return ns


def make_inputs(seed=11):
    g = torch.Generator().manual_seed(seed)
    faces = torch.stack([torch.randperm(V, generator=g)[:3] for _ in range(F)]).int()
    verts = torch.randn(V, 3, generator=g)
    with_gaussians = torch.tensor([f for f in range(F) if f not in NO_GAUSSIANS])
    cells = with_gaussians[torch.randint(0, len(with_gaussians), (P,), generator=g)]
    cells[:len(with_gaussians)] = with_gaussians[torch.randperm(len(with_gaussians), generator=g)][:P]
    sh_dc = 2.0 * torch.randn(P, 1, 3, generator=g)
    seen = torch.tensor([f for f in range(F) if f not in UNSEEN])
    images, p2fs, barys = [], [], []
    for v in range(N_VIEWS):
        # 4x4 blocks (the last row of blocks 4x... cut by H = 20) share a face; about a fifth of them are background
        blocks = seen[torch.randint(0, len(seen), (H // 4 + 1, W // 4 + 1), generator=g)]
        blocks[torch.rand(blocks.shape, generator=g) < 0.2] = -1
        p2f = blocks.repeat_interleave(4, 0).repeat_interleave(4, 1)[:H, :W].contiguous().int()
        # barycentrics: u, v >= 0 with u + v <= 1 (a few a hair outside the triangle), third = 1 - (u + v) in fp32
        uv = torch.rand(H, W, 2, generator=g)
        flip = uv.sum(-1) > 1
        uv[flip] = 1 - uv[flip]
        uv = uv + 1e-3 * (torch.rand(H, W, 2, generator=g) < 0.05) * torch.randn(H, W, 2, generator=g)
        bary = torch.cat([uv, 1. - uv.sum(dim=-1, keepdim=True)], -1)
        bary[p2f < 0] = torch.tensor([0., 0., 1.])
        img = torch.rand(H, W, 3, generator=g) * 1.4 - 0.2
        special = torch.rand(H, W, 3, generator=g)
        img[special < 0.02] = float("nan")
        img[(special >= 0.02) & (special < 0.03)] = float("inf")
        img[(special >= 0.03) & (special < 0.04)] = -float("inf")
        images.append(img)
        p2fs.append(p2f)
        barys.append(bary.contiguous())
    return dict(faces=faces, verts=verts, cells=cells, sh_dc=sh_dc, images=torch.stack(images),
                pix_to_face=torch.stack(p2fs), bary=torch.stack(barys))


def main():
    x = make_inputs()
    ns = reference_namespace([(x["pix_to_face"][v], x["bary"][v]) for v in range(N_VIEWS)])
    cams = _Cameras([SimpleNamespace(image_height=H, image_width=W)] * N_VIEWS)
    frosting = SimpleNamespace(
        device="cpu", nerfmodel=SimpleNamespace(training_cameras=cams),
        shell_base=_Meshes([x["verts"]], [x["faces"]]), _point_cell_indices=x["cells"], _sh_coordinates_dc=x["sh_dc"],
        render_image_gaussian_rasterizer=lambda camera_indices, **kw: x["images"][camera_indices].clone())
    save = {k: v.numpy() for k, v in x.items()}
    save["square_sizes"] = np.array(SQUARE_SIZES, np.int32)
    for sq in SQUARE_SIZES:
        out = ns["compute_textured_mesh_for_frosting_mesh"](frosting, square_size=sq, n_sh=0,
                                                            texture_with_gaussian_renders=True, bg_color=[0., 0., 0.],
                                                            use_occlusion_culling=False)
        save[f"texture_{sq}"] = out.textures.maps[0].numpy()
        save[f"verts_uvs_{sq}"] = out.textures.verts_uvs[0].numpy()
        save[f"faces_uvs_{sq}"] = out.textures.faces_uvs[0].numpy()
        assert out.verts[0] is x["verts"] and out.faces[0] is x["faces"]
    np.savez_compressed(os.path.join(HERE, "frosting_texture_bake.npz"), **save)
    print(len(save), "arrays", sum(v.nbytes for v in save.values()), "bytes")


if __name__ == "__main__":
    main()
