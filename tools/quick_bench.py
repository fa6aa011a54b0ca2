"""Developer timing script (not the contract bench): per-stage CUDA-event timings of frosting_b200 vs
the compiled reference on random scenes, alternating, median of 10 after 3 warm-up rounds.
Usage: python tools/quick_bench.py [P W H D]"""
import sys
import os
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import frosting_b200 as fb
from frosting_b200 import scenes
from oracle import refdgr
from tools import timing


def main():
    P, W, H, D = (int(x) for x in (sys.argv[1:5] if len(sys.argv) >= 5 else (500_000, 800, 800, 3)))
    dev = torch.device("cuda:0")
    cam = scenes.make_camera(W, H, device=dev)
    g = scenes.random_gaussians(P, cam, 1234, device=dev)
    rs = scenes.settings_for(cam, D, device=dev)
    cot = torch.randn(3, H, W, device=dev)
    kw = dict(shs=g["shs"], scales=g["scales"], rotations=g["rotations"])

    def mine_fwd():
        with torch.no_grad():
            return fb.GaussianRasterizer(rs)(means3D=g["means3D"], means2D=None, opacities=g["opacities"], **kw)

    leaves = {k: g[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "shs", "scales", "rotations")}

    def mine_fb():
        for v in leaves.values():
            v.grad = None
        m2 = torch.zeros(P, 3, device=dev, requires_grad=True)
        c, _ = fb.GaussianRasterizer(rs)(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"],
                                         shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"])
        c.backward(cot)

    def ref_fwd():
        return refdgr.forward(rs, g["means3D"], g["opacities"], **kw)

    def ref_fb():
        f = refdgr.forward(rs, g["means3D"], g["opacities"], **kw)
        return refdgr.backward(rs, f, g["means3D"], cot, **kw)

    st = fb.forward_with_state(rs, g["means3D"], g["opacities"], **kw)
    R = st["num_rendered"]
    print(f"P={P} {W}x{H} D={D} R={R} R/P={R / P:.2f} visible={(st['radii'] > 0).float().mean().item():.3f} "
          f"max_tile={int(st['tile_count'].max())}")
    routes = {"mine_fwd": mine_fwd, "mine_fb": mine_fb}
    if refdgr.available():
        routes.update(ref_fwd=ref_fwd, ref_fb=ref_fb)
    t = {k: s["median_ms"] for k, s in timing.alternate(routes, 10, 3)[0].items()}
    t_mf, t_mfb = t["mine_fwd"], t["mine_fb"]
    print(f"mine: fwd {t_mf:.3f} ms  fwd+bwd {t_mfb:.3f} ms  ({1000 / t_mfb:.1f} fps)")
    if refdgr.available():
        t_rf, t_rfb = t["ref_fwd"], t["ref_fb"]
        print(f"ref : fwd {t_rf:.3f} ms  fwd+bwd {t_rfb:.3f} ms  ({1000 / t_rfb:.1f} fps)")
        print(f"speedup fwd {t_rf / t_mf:.2f}x  fwd+bwd {t_rfb / t_mfb:.2f}x")


if __name__ == "__main__":
    main()
