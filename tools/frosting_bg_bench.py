"""Frosting mode with background Gaussians against the route a user had without it.

    python tools/frosting_bg_bench.py [--n-bg 0 500000] [--iters 20] [--warmup 3]

Scene: the C3 frosting layer (2 M mesh-bound Gaussians, ~1 M-face shell, 1920x1080, SH degree 3, ring camera at radius 6,
occlusion lookup) plus `n_bg` background Gaussians from `scenes.frosting_layer(..., n_background=n_bg)`.  Per iteration,
forward + loss + backward, timed with CUDA events, the two routes alternating:
  (a) `frosting_render` with the six bg_* parameters (one frame, attributes built in preprocess, parameter gradients
      written by the per-Gaussian backward);
  (b) `frosting_attributes_fused` for the mesh rows, Frosting's torch bg_* chain (`scenes.frosting_background_attributes`),
      `torch.cat`, `GaussianRasterizer(face_visibility=...)`, autograd back through the chain.
Checks that (a) and (b) agree: radii (all but ~1e-3 of the Gaussians) and image (statistical, the torch chain's
attributes differ by an ulp).  Prints the card and its power limit with the numbers.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frosting_b200 as fb                       # noqa: E402
from frosting_b200 import scenes                 # noqa: E402
from frosting_b200.frosting_render import BG_KEYS, MESH_KEYS   # noqa: E402
from tools import timing                                       # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-bg", type=int, nargs="+", default=[0, 500_000])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n-mesh", type=int, default=2_000_000)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    W, H = 1920, 1080
    cam0 = scenes.make_camera(W, H)
    cam = scenes.ring_cameras(8, W, H, radius=6.0, device=dev)[0]
    rs = scenes.settings_for(cam, 3, device=dev)
    gpu = timing.card()
    result = {"card": gpu, "gpu": gpu["name"], "power_limit": gpu["power_limit"], "n_mesh": args.n_mesh, "runs": []}
    for n_bg in args.n_bg:
        params, mesh = scenes.frosting_layer(args.n_mesh, cam0, 1237, n_faces_target=max(1000, args.n_mesh // 2),
                                             n_background=n_bg)
        params = {k: v.to(dev).requires_grad_(True) for k, v in params.items()}
        mesh = {k: v.to(dev) for k, v in mesh.items()}
        _, fv, _ = fb.rasterize_mesh(mesh["verts"], mesh["faces"], cam.full_proj_transform, H, W, mark_last_on_bg=True)
        cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(3)).to(dev)

        def route_a():
            color, radii = fb.frosting_render(params, mesh, rs, face_visible=fv)
            (color * cot).sum().backward()
            return color, radii

        def route_b():
            a = fb.frosting_attributes_fused({k: params[k] for k in MESH_KEYS}, mesh, face_visible=fv)
            if n_bg:
                b = scenes.frosting_background_attributes(params)
                a = {k: torch.cat([a[k], b[k]]) for k in a}
            P = a["means3D"].shape[0]
            color, radii = fb.GaussianRasterizer(rs)(
                means3D=a["means3D"], means2D=torch.zeros(P, 3, device=dev), opacities=a["opacities"], shs=a["shs"],
                scales=a["scales"], rotations=a["rotations"], face_visibility=(fv, mesh["cells"]))
            (color * cot).sum().backward()
            return color, radii

        def clear_grads():
            for p in params.values():
                p.grad = None

        times, outs = timing.alternate({"a_frosting_render": route_a, "b_torch_cat_rasterizer": route_b}, args.iters,
                                       args.warmup, before=clear_grads)
        (ca, ra), (cb, rb) = outs["a_frosting_render"], outs["b_torch_cat_rasterizer"]
        d = (ca - cb).abs()
        check = {"radii_mismatch_frac": (ra != rb).float().mean().item(),
                 "image_px_over_1e-4_frac": (d > 1e-4).float().mean().item(), "image_max_abs_diff": d.max().item()}
        check["ok"] = check["radii_mismatch_frac"] < 1e-3 and check["image_px_over_1e-4_frac"] < 1e-3 and \
            check["image_max_abs_diff"] < 2e-2
        run = {"n_bg": n_bg, "rendered": int((ra > 0).sum()), "rendered_bg": int((ra[args.n_mesh:] > 0).sum()),
               "check": check, **times}
        run["speedup_b_over_a"] = run["b_torch_cat_rasterizer"]["median_ms"] / run["a_frosting_render"]["median_ms"]
        result["runs"].append(run)
        print(json.dumps(run), flush=True)
        del params, mesh, outs
        torch.cuda.empty_cache()
    timing.emit(result)


if __name__ == "__main__":
    main()
