"""SuGaR's depth-normal consistency (csrc/sugar_dn.cu) in the coarse `dn_consistency` trainer's step, against the
reference's structure on this project's rasterizer.

    python tools/sugar_dn_bench.py [--sizes 1000000 3000000] [--steps 30] [--warmup 5] [--out F]

Workload: `scenes.sugar_scene` at each size with seeded degree-3 SH coefficients, 1920x1080, `make_camera`'s default
camera, a seeded ground-truth image.  Routes, alternating within each step, each timed with CUDA events around forward
+ backward (autograd over every Gaussian parameter):
  (a) the colour frame + L1-DSSIM alone;
  (b) (a) plus the fused term: depth_normal_features as three extra channels of the same frame, then
      0.05 x depth_normal_consistency;
  (c) (a) plus the reference's structure: the features in torch, a second rasterizer call with them as colors_precomp
      and background 0, and the float32 torch loss (torch_reference_loss, the reference's lines).
Reported: medians and p10/p90 over `--steps` steps after `--warmup`, (b) - (a) and (c) - (a) from the medians, the card
and its power limit.  Then, in a separate run under the torch profiler (CUDA activity), the device time per step of each
kernel of (a) and of (b): the features kernels, the loss kernels, and the blend kernels of both, whose difference is the
E = 3 extra-channel instance's cost over the colour-only one.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frosting_b200 as fb                       # noqa: E402
from frosting_b200 import scenes, sugar_dn       # noqa: E402
from tools import timing                         # noqa: E402


GROUPS = {"features": ("dn_features_kernel", "dn_features_bwd_kernel"),
          "loss": ("dn_loss_fwd_kernel", "dn_loss_bwd_kernel"),
          "blend": ("render_fwd_pair_kernel", "render_bwd_t16_kernel", "extra_grad_kernel")}


def workload(P, dev):
    sc = {k: v.to(dev) for k, v in scenes.sugar_scene(P, 1, K=1).items() if k != "knn_idx"}
    gen = torch.Generator().manual_seed(2)
    shs = (0.3 * torch.randn(P, 16, 3, generator=gen)).to(dev)
    gt = torch.rand(3, 1080, 1920, generator=gen).to(dev)
    rs = scenes.settings_for(scenes.make_camera(1920, 1080, device=dev), 3, device=dev)
    rs0 = rs._replace(bg=torch.zeros(3, device=dev))
    leaves = {k: v.clone().requires_grad_(True) for k, v in dict(sc, shs=shs).items()}

    def frame(**kw):
        m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
        return fb.GaussianRasterizer(rs)(means3D=leaves["points"], means2D=m2, opacities=leaves["strengths"],
                                         shs=leaves["shs"], scales=leaves["scaling"], rotations=leaves["quaternions"],
                                         **kw)

    def grad(loss):
        torch.autograd.grad(loss, list(leaves.values()))

    def route_a():
        rgb, _ = frame()
        grad(fb.l1_dssim_loss(rgb, gt))

    def route_b():
        feats = fb.depth_normal_features(leaves["points"], leaves["scaling"], leaves["quaternions"], rs)
        rgb, _, dn = frame(extra_features=feats)
        grad(fb.l1_dssim_loss(rgb, gt) + 0.05 * fb.depth_normal_consistency(dn, rs))

    def route_c():
        rgb, _ = frame()
        feats = sugar_dn.torch_reference_features(leaves["points"], leaves["scaling"], leaves["quaternions"],
                                                  rs.viewmatrix, rs.campos)
        m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
        dn, _ = fb.GaussianRasterizer(rs0)(means3D=leaves["points"], means2D=m2, opacities=leaves["strengths"],
                                           colors_precomp=feats, scales=leaves["scaling"],
                                           rotations=leaves["quaternions"])
        loss = fb.l1_dssim_loss(rgb, gt) + 0.05 * sugar_dn.torch_reference_loss(dn, rs.viewmatrix, rs.projmatrix)
        grad(loss)

    def losses():
        with torch.no_grad():
            feats = fb.depth_normal_features(sc["points"], sc["scaling"], sc["quaternions"], rs)
            _, _, dn = fb.GaussianRasterizer(rs)(
                means3D=sc["points"], means2D=torch.zeros(P, 3, device=dev), opacities=sc["strengths"], shs=shs,
                scales=sc["scaling"], rotations=sc["quaternions"], extra_features=feats)
            return (float(fb.depth_normal_consistency(dn, rs)),
                    float(sugar_dn.torch_reference_loss(dn.double(), rs.viewmatrix.double(), rs.projmatrix.double())))

    return route_a, route_b, route_c, losses


def run(P, steps, warmup, dev):
    w = workload(P, dev)
    routes, losses = dict(zip("abc", w[:3])), w[3]
    s = timing.alternate(routes, steps, warmup)[0]
    out = {"P": P, "W": 1920, "H": 1080, "routes": s,
           "b_minus_a_ms": round(s["b"]["median_ms"] - s["a"]["median_ms"], 4),
           "c_minus_a_ms": round(s["c"]["median_ms"] - s["a"]["median_ms"], 4)}
    ours, f64 = losses()
    out["dn_loss"] = {"cuda": ours, "float64_reference": f64}
    ka, ga = timing.kernel_times(routes["a"], steps, GROUPS)
    kb, gb = timing.kernel_times(routes["b"], steps, GROUPS)
    out["profile_a"], out["profile_b"] = ka, kb
    out["groups_ms"] = {"features": gb["features"], "loss": gb["loss"], "blend_a": ga["blend"], "blend_b": gb["blend"],
                        "blend_extra": round(gb["blend"] - ga["blend"], 4)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sugar_dn_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": timing.card(), "torch": torch.__version__, "runs": []}
    for P in a.sizes:
        r = run(P, a.steps, a.warmup, dev)
        print(json.dumps(r), flush=True)
        res["runs"].append(r)
    timing.emit(res, a.out)


if __name__ == "__main__":
    main()
