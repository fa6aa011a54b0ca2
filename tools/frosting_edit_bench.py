"""One frame of an animated Frosting scene: the CUDA edit path against the torch chain a user runs without it.

    python tools/frosting_edit_bench.py [--n-bg 0 500000] [--iters 10] [--warmup 3] [--rescaling median]
                                        [--adaptation simple|complex] [--bones 0]

Scene: the C3 frosting layer (2 M mesh-bound Gaussians, ~1 M-face shell, 1920x1080, SH degree 3, ring camera at radius
6) plus `n_bg` background Gaussians, made editable (`--adaptation`, simple by default; 70 % of the faces edited); every
frame bends the sphere by a different twist and squash (`scenes.deform_base` at a frame-dependent strength).  Per frame, timed with
CUDA events, the two routes alternating:
  (a) `frosting_render_edited` (csrc/frosting_edit.cu: shell + tables, attributes with SH colours; then the rasterizer);
  (b) `scenes.edited_frosting_attributes` -- the torch restatement of the reference's per-frame chain (shell with
      pytorch3d-style normals, rotations, rescaling, deformation drop, SH colours in torch at rotated directions; with
      `--adaptation complex` the cell transforms and T_frame[cell] C, C solved once before the frames as make_editable
      does) -- then the same rasterizer with colors_precomp.  The reference's `.median().item()` host read-backs are
      not in it.
With `--bones N` (N > 0) the frames come from a rig instead (`scenes.skinned_rig`: a chain of N bones up the sphere,
12 frames of pose tracks) and each route poses the base mesh inside its timed frame: (a) `FrostingSkin.pose`
(csrc/frosting_skin.cu), (b) `scenes.skin_vertices`, the torch restatement of the reference's apply_poses_to_scene
(per bone: torch.inverse with its host synchronisation, two transform_points, a float64 multiply, an index +=).  The
skinning stage alone is then timed the same way, alternating.
Reports the median of `--iters` frames per route, the max image difference and radii agreement between the routes,
and the card and its power limit.
"""
import argparse
import itertools
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frosting_b200 as fb                       # noqa: E402
from frosting_b200 import rasterizer as R        # noqa: E402
from frosting_b200 import scenes                 # noqa: E402
from tools import timing                         # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-bg", type=int, nargs="+", default=[0, 500_000])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--n-mesh", type=int, default=2_000_000)
    ap.add_argument("--rescaling", default="median", choices=["median", "triangle"])
    ap.add_argument("--adaptation", default="simple", choices=["simple", "complex"])
    ap.add_argument("--bones", type=int, default=0)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    W, H = 1920, 1080
    cam = scenes.ring_cameras(8, W, H, radius=6.0, device=dev)[0]
    rs = scenes.settings_for(cam, 3, device=dev)
    gpu = timing.card()
    result = {"card": gpu, "gpu": gpu["name"], "power_limit": gpu["power_limit"], "n_mesh": args.n_mesh,
              "rescaling": args.rescaling, "adaptation": args.adaptation, "bones": args.bones,
              "runs": []}
    e = torch.Tensor([])
    for n_bg in args.n_bg:
        params, mesh = scenes.frosting_layer(args.n_mesh, scenes.make_camera(W, H), 1237,
                                             n_faces_target=max(1000, args.n_mesh // 2), n_background=n_bg, device=dev)
        V, F = mesh["verts"].shape[0], mesh["faces"].shape[0]
        g = torch.Generator().manual_seed(4)
        inner_dist = (-0.02 * (1 + 0.2 * torch.rand(V, generator=g))).to(dev)
        outer_dist = (0.02 * (1 + 0.2 * torch.rand(V, generator=g))).to(dev)
        em = (torch.rand(F, generator=g) < 0.7).to(dev)
        quats = torch.cat([params["quats"], params["bg_quats"]]) if n_bg else params["quats"]
        orig = torch.nn.functional.normalize(quats + 0.2 * torch.randn(quats.shape, generator=g).to(dev), dim=-1)
        canonical = None
        if args.adaptation == "simple":
            edit = fb.FrostingEdit(mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist, edition_mask=em,
                                   thickness_rescaling=args.rescaling)
        else:
            edit = fb.FrostingEditComplex(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist,
                                          edition_mask=em, thickness_rescaling=args.rescaling)
            with torch.no_grad():
                canonical, _ = scenes.complex_canonical_transforms(params, mesh["verts"], mesh["faces"], mesh["cells"],
                                                                   em, args.rescaling)

        if args.bones:
            package, ref_indices = scenes.skinned_rig(mesh["verts"], args.bones, 12)
            skin = fb.FrostingSkin(package, ref_indices, V, dev)
            buf_a, buf_b = mesh["verts"].clone(), mesh["verts"].clone()
            frame = lambda i: i                       # a frame index: each route poses the mesh itself
            pose_a = lambda i: skin.pose(i, buf_a)
            pose_b = lambda i: scenes.skin_vertices(package, ref_indices, i, buf_b)
        else:                                         # the deformed mesh: an input made outside the timed window
            frame = lambda i: scenes.deform_base(mesh["verts"], 0.4 + 0.05 * (i % 12))
            pose_a = pose_b = lambda verts: verts

        x = {}                                        # the frame every route of a step renders

        def route_a():
            return fb.frosting_render_edited(params, edit, pose_a(x["frame"]), rs, orig_quats=orig)

        def route_b():
            a = scenes.edited_frosting_attributes(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist,
                                                  outer_dist, pose_b(x["frame"]), rs.campos, 3, edition_mask=em,
                                                  thickness_rescaling=args.rescaling, orig_quats=orig,
                                                  adaptation=args.adaptation, canonical=canonical)
            color, radii, _, _ = R._launch_forward(a["means3D"], e, a["colors_precomp"], a["opacities"], a["scales"],
                                                   a["rotations"], e, rs, None)
            return color, radii

        def timed(routes):
            calls = itertools.count()

            def next_frame():       # made outside the timed window: frames 0, 1, ... over the warm-up, then from 0 again
                i = next(calls) // len(routes)
                x["frame"] = frame(i if i < args.warmup else i - args.warmup)

            with torch.no_grad():
                return timing.alternate(routes, args.iters, args.warmup, before=next_frame)

        stats, outs = timed({"a_frosting_render_edited": route_a, "b_torch_chain_rasterizer": route_b})
        (ca, ra), (cb, rb) = outs["a_frosting_render_edited"], outs["b_torch_chain_rasterizer"]
        run = {"n_bg": n_bg, "rendered": int((ra > 0).sum()), "image_max_abs_diff": (ca - cb).abs().max().item(),
               "image_px_over_1e-4_frac": ((ca - cb).abs() > 1e-4).float().mean().item(),
               "radii_agree_frac": (ra == rb).float().mean().item(), **stats}
        run["speedup_b_over_a"] = run["b_torch_chain_rasterizer"]["median_ms"] / run["a_frosting_render_edited"]["median_ms"]
        if args.bones:
            skin_stats, skin_outs = timed({"a_skin_cuda": lambda: pose_a(x["frame"]),
                                           "b_skin_torch": lambda: pose_b(x["frame"])})
            run["skin"] = dict(skin_stats, max_abs_diff=(skin_outs["a_skin_cuda"] - skin_outs["b_skin_torch"]).abs().max().item(),
                               speedup_b_over_a=skin_stats["b_skin_torch"]["median_ms"] / skin_stats["a_skin_cuda"]["median_ms"])
        result["runs"].append(run)
        print(json.dumps(run), flush=True)
        del params, mesh, outs, edit, canonical, pose_a, pose_b
        torch.cuda.empty_cache()
    timing.emit(result)


if __name__ == "__main__":
    main()
