"""The texture bake of a trained Frosting model: the CUDA bake against the torch route a user runs without it.

    python tools/texture_bench.py [--cameras 64] [--square-size 8] [--iters 3] [--warmup 1] [--obj-dir DIR]

Scene: the C3 frosting layer (2 M mesh-bound Gaussians, ~1 M-face base mesh, 1920x1080), `--cameras` ring cameras at
radius 6, square size 8 (T = 5664: 32 M texels).  Routes, alternating, each timed with CUDA events around a whole bake:
  (a) `compute_textured_mesh` (csrc/texture.cu): per view rasterize_mesh, `render_view` at SH degree 0, mesh_bary,
      add_view; then finish;
  (b) per view the same render (`render_view`, SH degree 0) and MeshRasterizer (the prepass plus mesh._barycentrics in torch), then
      `scenes.bake_texture_torch` on the GPU over the collected views -- texture.py's scatter and fill in torch.
Then the stages of (a) alone over views rendered beforehand, each median over the views of `--iters` passes: mesh_bary
per view, add_view per view, finish (the fill), and the once-per-bake set-up (TextureBaker: accumulators, CSR, SH
colours).  With `--obj-dir`, `write_textured_obj` of route (a)'s result is timed on the host (OBJ + MTL + PNG).
Reports the medians, the agreement of the two routes' textures, and the card and its power limit.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frosting_b200 as fb                       # noqa: E402
from frosting_b200 import scenes                 # noqa: E402
from frosting_b200.mesh import MeshRasterizer, rasterize_mesh   # noqa: E402
from frosting_b200.texture import _settings, render_view      # noqa: E402


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def stats(t):
    t = sorted(t)
    return {"median_ms": t[len(t) // 2], "min_ms": t[0], "max_ms": t[-1]}


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return out, e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, default=64)
    ap.add_argument("--square-size", type=int, default=8)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--n-mesh", type=int, default=2_000_000)
    ap.add_argument("--obj-dir", default=None, help="time write_textured_obj into this directory (a temporary one "
                                                    "if 'tmp')")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    W, H = 1920, 1080
    sq = args.square_size
    params, mesh = scenes.frosting_layer(args.n_mesh, scenes.make_camera(W, H), 1237,
                                         n_faces_target=max(1000, args.n_mesh // 2), device=dev)
    cams = scenes.ring_cameras(args.cameras, W, H, radius=6.0, device=dev)
    verts, faces = mesh["verts"], mesh["faces"]
    bg = torch.zeros(3, device=dev)
    F = faces.shape[0]
    result = {"gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "n_mesh": args.n_mesh,
              "n_faces": F, "cameras": args.cameras, "image": [W, H], "square_size": sq,
              "texture_size": sq * int(math.sqrt(F // 2 + 1) + 1)}

    def route_a():
        return fb.compute_textured_mesh(params, mesh, cams, square_size=sq)["texture_map"]

    def route_b():
        rasterizer = MeshRasterizer(cameras=cams)
        images, p2fs, barys = [], [], []
        for i, cam in enumerate(cams):
            img = render_view(params, mesh, _settings(cam, 0, bg, dev))
            frag = rasterizer((verts, faces), cam_idx=i)
            images.append(img.permute(1, 2, 0))
            p2fs.append(frag.pix_to_face.view(H, W))
            barys.append(frag.bary_coords.view(H, W, 3))
        return scenes.bake_texture_torch(F, mesh["cells"], params["sh_dc"], sq, images, p2fs, barys)[2]

    times = {"a_compute_textured_mesh": [], "b_torch_bake": []}
    outs = {}
    with torch.no_grad():
        for i in range(args.warmup + args.iters):
            for name, fn in (("a_compute_textured_mesh", route_a), ("b_torch_bake", route_b)):
                outs.pop(name, None)
                outs[name], ms = timed(fn)
                if i >= args.warmup:
                    times[name].append(ms)
        for name, t in times.items():
            result[name] = stats(t)
        result["speedup_b_over_a"] = result["b_torch_bake"]["median_ms"] / result["a_compute_textured_mesh"]["median_ms"]
        ta, tb = outs["a_compute_textured_mesh"], outs["b_torch_bake"]
        result["texels_equal_frac"] = (ta == tb).all(dim=-1).float().mean().item()
        result["texture_max_abs_diff"] = (ta - tb).abs().max().item()
        del outs, tb
        torch.cuda.empty_cache()

        # stages of route (a) over views rendered beforehand
        views = []
        for cam in cams:
            p2f, _, _ = rasterize_mesh(verts, faces, cam.full_proj_transform, H, W)
            img = render_view(params, mesh, _settings(cam, 0, bg, dev))
            views.append((cam, p2f, img.permute(1, 2, 0).contiguous()))
        stage = {"setup": [], "mesh_bary": [], "add_view": [], "finish": []}
        for i in range(args.warmup + args.iters):
            baker, ms = timed(lambda: fb.TextureBaker(faces, mesh["cells"], params["sh_dc"], verts.shape[0], sq))
            keep = i >= args.warmup
            if keep:
                stage["setup"].append(ms)
            for cam, p2f, img in views:
                bary, ms = timed(lambda: fb.mesh_bary(verts, faces, cam.full_proj_transform, p2f))
                if keep:
                    stage["mesh_bary"].append(ms)
                _, ms = timed(lambda: baker.add_view(img, p2f, bary))
                if keep:
                    stage["add_view"].append(ms)
            (_, _, tex), ms = timed(baker.finish)
            if keep:
                stage["finish"].append(ms)
            del baker, tex
        result["stages"] = {k: stats(v) for k, v in stage.items()}
        result["hit_pixels_per_view"] = sum(int((p2f >= 0).sum()) for _, p2f, _ in views) / len(views)
        del views

        if args.obj_dir:
            out = fb.compute_textured_mesh(params, mesh, cams, square_size=sq)
            with tempfile.TemporaryDirectory() as tmp:
                d = tmp if args.obj_dir == "tmp" else args.obj_dir
                os.makedirs(d, exist_ok=True)
                t0 = time.perf_counter()
                paths = fb.write_textured_obj(os.path.join(d, "frosting_textured.obj"), **out)
                result["write_obj_s"] = time.perf_counter() - t0
                result["obj_bytes"] = {os.path.basename(p): os.path.getsize(p) for p in paths}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
