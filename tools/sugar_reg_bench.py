"""SuGaR's SDF regulariser (csrc/sugar_reg.cu) against the reference's torch route, on the coarse trainer's workload.

    python tools/sugar_reg_bench.py [--sizes 1000000 3000000] [--samples 1000000] [--steps 30] [--warmup 5] [--out F]

Scenes: `scenes.sugar_scene` (flat Gaussians on a bumpy sphere, 10 % volumetric stragglers, K = 16 cKDTree neighbours,
self first) at each size; the sampling mask is `radii > 0` of one drop-in rasterizer frame at 1920x1080 (SH degree 3),
the samples `sample_in_gaussians(mask, --samples)`.  Routes, alternating within each step, each timed with CUDA events:
  (a) `sdf_regularization`, forward + backward (autograd.grad of 0.2 est + 0.2 nrm);
  (b) `torch_reference` in float32 on the GPU, forward + backward (the reference's arithmetic and kernels);
  the sampler alone; one rasterizer frame (forward + backward) on the same scene, for scale;
  and the op's own pieces: forward without gradient, forward with gradient (the per-pair pass also differentiating),
  backward (the per-Gaussian chain kernel).
These are call times: CUDA events around the Python call, host work included.  Then, in a separate run under the
torch profiler (CUDA activity), the device time of each of the op's kernels over `--steps` steps of forward with
gradient + backward and of forward without gradient (inputs detached, so the gradient pass is not asked for).
Medians and p10/p90 over `--steps` timed steps after `--warmup`; each route's peak extra memory; the agreement of (a)
with (b); the card and its power limit; the sample kernel's bytes over its own device time.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frosting_b200 as fb                       # noqa: E402
from frosting_b200 import scenes, sugar          # noqa: E402
from tools import timing                         # noqa: E402

LEAVES = ("points", "scaling", "quaternions", "strengths")


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


KERNELS = ("sugar_record_kernel", "sugar_sample_kernel", "sugar_terms_kernel", "sugar_chain_kernel")


def kernel_name(key):
    for n in KERNELS:
        if n in key:
            if n == "sugar_sample_kernel":       # the template's `grad` argument, demangled or not
                return n + ("<grad>" if ("true>" in key or "Lb1E" in key) else "<nograd>")
            return n
    return "memset" if "Memset" in key else key[:80]


def by_kernel(kernels):
    """`timing.kernel_times`' table with the op's kernels and the memsets each summed under one name."""
    out = {}
    for key, ms in kernels.items():
        out[kernel_name(key)] = round(out.get(kernel_name(key), 0.0) + ms, 4)
    return out


def workload(P, N, dev):
    sc = scenes.sugar_scene(P, 1, K=16)
    knn = sc.pop("knn_idx")
    sc = {k: v.to(dev) for k, v in sc.items()}
    cam = scenes.make_camera(1920, 1080, device=dev)
    rs = scenes.settings_for(cam, 3, device=dev)
    shs = (0.3 * torch.randn(P, 16, 3, generator=torch.Generator().manual_seed(2))).to(dev)
    raster = fb.GaussianRasterizer(rs)
    leaves = {k: v.clone().requires_grad_(True) for k, v in sc.items()}
    shs_l = shs.clone().requires_grad_(True)

    def frame():
        m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
        color, radii = raster(means3D=leaves["points"], means2D=m2, opacities=leaves["strengths"], shs=shs_l,
                              scales=leaves["scaling"], rotations=leaves["quaternions"])
        color.sum().backward()
        return radii

    with torch.no_grad():
        _, radii = raster(means3D=sc["points"], means2D=torch.zeros(P, 3, device=dev), opacities=sc["strengths"],
                          shs=shs, scales=sc["scaling"], rotations=sc["quaternions"])
    return sc, sugar.SugarNeighbours(knn.to(dev)), radii > 0, frame


def run(P, N, steps, warmup, dev):
    sc, nb, mask, frame = workload(P, N, dev)
    torch.manual_seed(0)
    idx, eps = sugar.sample_in_gaussians(mask, N)
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]

    def ours():
        est, nrm = sugar.sdf_regularization(*leaves, nb, idx, eps)
        return (est, nrm), torch.autograd.grad(0.2 * est + 0.2 * nrm, leaves)

    def ref():
        est, nrm = sugar.torch_reference(*leaves, nb.knn_idx.long(), idx, eps)
        return (est, nrm), torch.autograd.grad(0.2 * est + 0.2 * nrm, leaves)

    def fwd_nograd():
        with torch.no_grad():
            return sugar.sdf_regularization(*leaves, nb, idx, eps)

    held = {}

    def fwd_grad():
        held["terms"] = sugar.sdf_regularization(*leaves, nb, idx, eps)
        return held["terms"]

    def bwd():                           # the backward alone, over the forward the route before it made
        est, nrm = held.pop("terms")
        return torch.autograd.grad(0.2 * est + 0.2 * nrm, leaves)

    routes = {"cuda_fwd_bwd": ours, "torch_fwd_bwd": ref, "sampler": lambda: sugar.sample_in_gaussians(mask, N),
              "raster_frame": frame, "cuda_fwd_nograd": fwd_nograd, "cuda_fwd_grad": fwd_grad, "cuda_bwd": bwd}
    call_times = timing.alternate(routes, steps, warmup)[0]
    (to, go), mem_ours = peak(ours)
    (tr, gr), mem_ref = peak(ref)
    agree = {"terms_rel": [abs(float(a.detach() - b.detach())) / max(abs(float(b.detach())), 1e-30) for a, b in zip(to, tr)],
             "grad_max_rel": {k: float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
                              for k, a, b in zip(LEAVES, go, gr)}}
    detached = [l.detach() for l in leaves]

    def step_grad():
        est, nrm = sugar.sdf_regularization(*leaves, nb, idx, eps)
        torch.autograd.grad(0.2 * est + 0.2 * nrm, leaves)

    kt_grad = by_kernel(timing.kernel_times(step_grad, steps)[0])
    kt_nograd = by_kernel(timing.kernel_times(lambda: sugar.sdf_regularization(*detached, nb, idx, eps), steps)[0])
    M, K = int(mask.sum()), nb.K
    # bytes of the per-pair pass (the with-gradient forward): per pair one 80-byte record gather and five 16-byte
    # vector reductions; per sample the draws (20 B), the owner's quaternion, scales, record and table row, and five
    # owner reductions.  DRAM-minimal bytes: every input, record and accumulator once.
    pair_bytes = N * K * (80 + 5 * 16) + N * (20 + 16 + 12 + 80 + 4 * K + 5 * 16)
    dram_min = P * (12 + 12 + 16 + 4 + 4 * K + 80 + 128 + 44) + N * 20
    ms_pairs = kt_grad["sugar_sample_kernel<grad>"]
    return {"P": P, "K": K, "N": N, "masked": M,
            "call_times": call_times,
            "kernels_fwd_grad_plus_bwd_ms": kt_grad, "kernels_fwd_nograd_ms": kt_nograd,
            "peak_extra_bytes": {"cuda": mem_ours, "torch": mem_ref},
            "agreement": agree,
            "sample_kernel_grad_gathered_bytes": pair_bytes,
            "sample_kernel_grad_gathered_GBps": round(pair_bytes / ms_pairs / 1e6, 1),
            "dram_min_bytes": dram_min, "dram_min_GBps_over_sample_kernel": round(dram_min / ms_pairs / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sugar_reg_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": timing.card(), "torch": torch.__version__, "runs": []}
    for P in a.sizes:
        r = run(P, a.samples, a.steps, a.warmup, dev)
        print(json.dumps(r), flush=True)
        res["runs"].append(r)
    timing.emit(res, a.out)


if __name__ == "__main__":
    main()
