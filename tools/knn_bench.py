"""knn_points (csrc/knn.cu) on the scenes SuGaR's and Frosting's neighbour tables are built over, K = 16.

    python tools/knn_bench.py [--steps 30] [--warmup 3] [--out F] [--no-profile]

Cases: `scenes.knn_scene("sugar", P)` at P = 200 k, 1 M and 3 M (SuGaR surface, 10 % stragglers, 1 % far background
Gaussians out to 10^4 surface spacings); C3's 2 M frosting-layer centres and C5's 6 M free Gaussians as
`camera_batch.build_workload` makes them; 1 M coincident points (the tie clause of the pruning).  Self queries, the
trainers' call.  Each case: median and p10/p90 of `--steps` calls timed with CUDA events after `--warmup`, the whole
Python call: allocation of the workspace and outputs, and the host read of the 4-byte non-finite flag (a round trip the
events enclose, so the times are upper bounds on the device work).  For context: scipy's cKDTree on the host up to 1 M
distinct points (workers=-1, build + query, the route users have without pytorch3d; one timed call) and, at 200 k, an
exhaustive chunked brute force in torch on the GPU (squared distances in matmul form + topk: every pair is scored, but
not with the contract's float expression, so not bit-exact), a stand-in for pytorch3d's O(P^2) kernel.  Then, in a
separate run under the torch profiler, the device time per kernel at 1 M.  The card's name, power limit and max SM
clock are read before and after the run.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frosting_b200 import camera_batch, knn_points, scenes     # noqa: E402
from tools import timing                                        # noqa: E402

K = 16


def workload_points(name):
    P, W, H, D, kind, seed = camera_batch.WORKLOADS[name]
    threads = torch.get_num_threads()
    torch.set_num_threads(camera_batch.SCENE_THREADS)
    try:
        cam = scenes.make_camera(W, H)
        if kind == "frosting":
            params, mesh = scenes.frosting_layer(P, cam, seed, n_faces_target=max(1000, P // 2), device="cpu")
            return scenes.frosting_attributes(params, mesh)["means3D"].contiguous()
        return scenes.random_gaussians(P, cam, seed, device="cpu")["means3D"].contiguous()
    finally:
        torch.set_num_threads(threads)


def brute_force(points, chunk=4096):
    """K nearest by matmul-form squared distance in torch, every pair scored, chunked over the queries (O(P^2))."""
    n2 = (points * points).sum(1)
    out = []
    for q in points.split(chunk):
        d = (q * q).sum(1)[:, None] + n2[None] - 2 * q @ points.T
        out.append(d.topk(K, dim=1, largest=False).indices)
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--cases", nargs="*", default=None, help="run only the cases whose name contains one of these")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    cases = [("sugar 200k", lambda: scenes.knn_scene("sugar", 200_000, 1)),
             ("sugar 1M", lambda: scenes.knn_scene("sugar", 1_000_000, 1)),
             ("sugar 3M", lambda: scenes.knn_scene("sugar", 3_000_000, 1)),
             ("C3 2M frosting centres", lambda: workload_points("c3")),
             ("C5 6M free Gaussians", lambda: workload_points("c5")),
             ("1M coincident", lambda: torch.full((1_000_000, 3), 0.5))]
    gpu = timing.card()
    res = {"card": gpu, "card (name, power limit, max SM clock)": ", ".join(gpu.values()), "K": K, "cases": {}}
    for name, make in cases:
        if a.cases is not None and not any(c in name for c in a.cases):
            continue
        pts = make()
        g = pts.to(dev)
        row = {"P": len(pts), **timing.alternate({"knn_points": lambda: knn_points(g, K=K)}, a.steps, a.warmup)[0]}
        if len(pts) <= 1_000_000 and "coincident" not in name:     # cKDTree cannot split coincident points: O(P^2)
            from scipy.spatial import cKDTree
            t = time.perf_counter()
            cKDTree(pts.double().numpy()).query(pts.double().numpy(), k=K, workers=-1)
            row["cKDTree_host_ms"] = round(1e3 * (time.perf_counter() - t), 1)
            row["host_cpus"] = os.cpu_count()
        if len(pts) <= 200_000:
            row.update(timing.alternate({"torch_brute_force": lambda: brute_force(g)}, 3, 1)[0])
        res["cases"][name] = row
        print(json.dumps({name: row}), flush=True)
        del g
        torch.cuda.empty_cache()
    if not a.no_profile:
        g = scenes.knn_scene("sugar", 1_000_000, 1).to(dev)
        res["profile_sugar_1M_per_call"], _ = timing.kernel_times(lambda: knn_points(g, K=K), a.steps)
        print(json.dumps({"profile_sugar_1M_per_call": res["profile_sugar_1M_per_call"]}), flush=True)
    timing.emit(res, a.out)


if __name__ == "__main__":
    main()
