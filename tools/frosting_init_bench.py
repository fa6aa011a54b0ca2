"""A Frosting layer's initial thickness (frosting_init.py, csrc/frosting_init.cu) at 1 M base vertices.

    python tools/frosting_init_bench.py [--verts 1000000] [--gaussians 2000000] [--steps 5] [--warmup 1] [--out F]

Scene: `scenes.frosting_init_scene` with --verts vertices and --gaussians SuGaR and as many 3DGS Gaussians.  Routes,
timed alternately with CUDA events after the warm-up, whole Python calls:
  initial_shell        the CUDA route: knn_points tables, two fb200_level_points calls;
  torch_float32        torch_initial_shell: the reference's chunked torch computation (2 M samples per pass) in float32,
                       with the same knn_points tables and the scenes restatements of pytorch3d's maths.
Reported: the times, each route's peak device memory above the scene, agreement (the share of vertices whose outer /
inner distances differ by more than 1e-5, and the largest difference), per-kernel device times of initial_shell under
the torch profiler, and the card (name, power limit, max SM clock) before and after.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frosting_b200 import initial_shell, scenes                     # noqa: E402
from frosting_b200.frosting_init import torch_initial_shell        # noqa: E402
from tools import timing                                            # noqa: E402

EXTENT = 4.0


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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    gpu = timing.card()
    sc = scenes.frosting_init_scene(a.verts, a.gaussians, a.gaussians, 0)
    sugar, gs = tuple(t.to(dev) for t in sc["sugar"]), tuple(t.to(dev) for t in sc["gs"])
    verts, faces = sc["verts"].to(dev), sc["faces"].to(dev)
    routes = {"initial_shell": lambda: initial_shell(sugar, gs, verts, faces, EXTENT),
              "torch_float32": lambda: torch_initial_shell(sugar, gs, verts, faces, EXTENT)}
    times, last = timing.alternate(routes, a.steps, a.warmup)
    del last
    outs, mem = {}, {}
    for name, fn in routes.items():
        outs[name], mem[name] = peak(fn)
    ours, ref = outs["initial_shell"], outs["torch_float32"]
    agree = {}
    for k in ("outer_dist", "inner_dist"):
        diff = (getattr(ours, k) - getattr(ref, k)).abs()
        agree[k] = {"share_over_1e-5": round((diff > 1e-5).double().mean().item(), 6), "max": diff.max().item()}
    res = {"card": gpu, "card (name, power limit, max SM clock)": ", ".join(gpu.values()), "verts": len(verts),
           "faces": len(faces), "sugar_gaussians": len(sugar[0]), "gs_gaussians": len(gs[0]), "times": times,
           "speedup_median": round(times["torch_float32"]["median_ms"] / times["initial_shell"]["median_ms"], 2),
           "peak_MiB": mem, "agreement": agree}
    del outs, ours, ref
    if not a.no_profile:
        res["profile_initial_shell"], _ = timing.kernel_times(lambda: initial_shell(sugar, gs, verts, faces, EXTENT),
                                                              a.steps)
    timing.emit(res, a.out)


if __name__ == "__main__":
    main()
