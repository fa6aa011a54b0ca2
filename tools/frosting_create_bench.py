"""Creating a Frosting layer (frosting_create.py, csrc/frosting_init.cu) from 1 M base vertices.

    python tools/frosting_create_bench.py [--verts 1000000] [--gaussians 2000000] [--n 2000000] [--steps 3] [--warmup 1]
                                          [--out F] [--no-profile]

Scene: `scenes.frosting_create_scene` with --verts vertices (about twice as many faces) and --gaussians SuGaR and as many
3DGS Gaussians, N = --n frosting Gaussians.  Routes, timed alternately with CUDA events after the warm-up, whole calls
on a generator of the same seed:
  create_frosting      the CUDA route: thickness, 20 trimming iterations, volumes, draws, sampling, scales, SH, background;
  torch_float32        torch_create_frosting: the reference's torch computation in float32 with knn_points tables.
Reported: the times, each route's peak device memory above the scene, agreement (trimmed distances, volumes, cells,
positions), per-kernel device times of create_frosting under the torch profiler with the trimming's share, and the card
(name, power limit, max SM clock) before and after.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frosting_b200 import scenes                                            # noqa: E402
from frosting_b200.frosting_create import _create, torch_create_frosting   # noqa: E402
from tools import timing                                                    # noqa: E402


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--verts", type=int, default=1_000_000)
    ap.add_argument("--gaussians", type=int, default=2_000_000)
    ap.add_argument("--n", type=int, default=2_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = timing.card()
    sc = scenes.frosting_create_scene(a.verts, a.gaussians, a.gaussians, 0)
    sugar = tuple(t.to(dev) for t in sc["sugar"])
    gs = {k: v.to(dev) for k, v in sc["gs_raw"].items()}
    verts, faces = sc["verts"].to(dev), sc["faces"].to(dev)
    kw = dict(spatial_extent=sc["spatial_extent"], camera_center=sc["camera_center"].to(dev), n_gaussians=a.n)
    gen = lambda: torch.Generator(dev).manual_seed(0)
    routes = {"create_frosting": lambda: _create(sugar, gs, verts, faces, generator=gen(), **kw),
              "torch_float32": lambda: torch_create_frosting(sugar, gs, verts, faces, generator=gen(), **kw)}
    times, last = timing.alternate(routes, a.steps, a.warmup)
    del last
    outs, mem = {}, {}
    for name, fn in routes.items():
        outs[name], mem[name] = peak(fn)
    (p, m, info), (rp, rm, rvol) = outs["create_frosting"], outs["torch_float32"]
    t = info["trimmed"]
    agree = {"trimmed_inner_verts_max": (m["inner"] - rm["inner"]).abs().max().item(),
             "trimmed_outer_verts_max": (m["outer"] - rm["outer"]).abs().max().item(),
             "stopped_sides": int((t.inner_stop < 20).sum() + (t.outer_stop < 20).sum()),
             "volumes_rel_max": ((info["volumes"] - rvol).abs() / rvol.abs().clamp_min(1e-30)).max().item(),
             "cells_equal_share": (m["cells"] == rm["cells"]).double().mean().item(),
             "bary_logits_max": (p["bary_logits"] - rp["bary_logits"]).abs().max().item(),
             "log_scales_max": (p["log_scales"] - rp["log_scales"]).abs().max().item(),
             "sh_rows_equal_share": (p["sh_dc"] == rp["sh_dc"]).all(-1).all(-1).double().mean().item(),
             "n_bg": int(p["bg_points"].shape[0]) if "bg_points" in p else 0}
    res = {"card": gpu, "card (name, power limit, max SM clock)": ", ".join(gpu.values()), "verts": len(verts),
           "faces": len(faces), "sugar_gaussians": len(sugar[0]), "gs_gaussians": len(gs["_xyz"]), "n": a.n,
           "times": times,
           "speedup_median": round(times["torch_float32"]["median_ms"] / times["create_frosting"]["median_ms"], 2),
           "peak_MiB": mem, "agreement": agree}
    del outs, p, m, info, rp, rm, rvol, t
    if not a.no_profile:
        res["profile_create_frosting"], res["profile_groups"] = timing.kernel_times(
            lambda: _create(sugar, gs, verts, faces, generator=gen(), **kw), a.steps,
            groups={"trim": ("trim_",), "knn": ("knn",), "level": ("level_",), "sample": ("sample_", "finish_",
                                                                                            "cell_volumes")})
    timing.emit(res, a.out)


if __name__ == "__main__":
    main()
