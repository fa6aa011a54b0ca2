"""Golden vectors for Frosting's BACKGROUND-Gaussian attribute chain, produced by EXECUTING the reference's own
property source, like make_frosting_attr_golden.py does for the mesh-bound Gaussians.

The properties bg_points, bg_strengths, bg_sh_coordinates, bg_scaling and bg_quaternions
(frosting_scene/frosting_model.py:801-876) are cut out of the reference file with `ast`, compiled UNMODIFIED into a stub
class and run with the flags of the reference's default for real scenes (use_background_gaussians=True,
use_background_sphere=False, scale_activation=torch.exp) on the background parameters of a small `scenes.frosting_layer`.

    python tests/golden/make_frosting_bg_attr_golden.py     # writes tests/golden/frosting_bg_attrs.npz

Stores the six background parameters (param_bg_*), the five outputs, cotangents and the autograd gradients w.r.t. every
parameter.  tests/test_frosting_background_cpu.py pins `scenes.frosting_background_attributes` to them;
tests/test_frosting_background_gpu.py pins the background attribute kernels.
"""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_dir      # noqa: E402
REF = os.path.join(reference_dir(), "frosting_scene", "frosting_model.py")
WANT = ("bg_points", "bg_strengths", "bg_sh_coordinates", "bg_scaling", "bg_quaternions")


def reference_background_properties():
    if not os.path.exists(REF):
        raise SystemExit(f"{REF} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
    src = open(REF).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "Frosting")
    lines = src.splitlines()
    chunks = []
    for n in cls.body:
        if isinstance(n, ast.FunctionDef) and n.name in WANT:
            first = min([d.lineno for d in n.decorator_list] + [n.lineno])
            chunks.append("\n".join(lines[first - 1:n.end_lineno]))
    assert len(chunks) == len(WANT), [c.split("def ")[1].split("(")[0] for c in chunks]
    ns = {"torch": torch}
    exec(compile("class RefBgProps:\n" + "\n\n".join(chunks) + "\n", REF, "exec"), ns)
    return ns["RefBgProps"]


def main():
    from frosting_b200 import scenes
    RefBgProps = reference_background_properties()
    cam = scenes.make_camera(160, 96)
    params, _ = scenes.frosting_layer(8, cam, 17, n_faces_target=64, n_background=256)
    leaf = {k: v.clone().requires_grad_(True) for k, v in params.items() if k.startswith("bg_")}
    m = RefBgProps()
    m.device, m.sh_levels = torch.device("cpu"), 4
    m.use_background_gaussians, m.use_background_sphere = True, False
    m.scale_activation = torch.exp
    m._bg_points = leaf["bg_points"]
    m._bg_opacities = leaf["bg_opacity_logits"].view(-1, 1)      # the reference keeps [n,1], this project [n]
    m._bg_sh_coordinates_dc, m._bg_sh_coordinates_rest = leaf["bg_sh_dc"], leaf["bg_sh_rest"]
    m._bg_scales, m._bg_quaternions = leaf["bg_log_scales"], leaf["bg_quats"]
    out = dict(means3D=m.bg_points, opacities=m.bg_strengths, scales=m.bg_scaling, rotations=m.bg_quaternions,
               shs=m.bg_sh_coordinates)
    g = torch.Generator().manual_seed(6)
    cots = {k: torch.randn(v.shape, generator=g) for k, v in out.items()}
    sum((out[k] * cots[k]).sum() for k in out).backward()
    save = {f"param_{k}": v.detach().numpy() for k, v in leaf.items()}
    save.update({f"out_{k}": v.detach().numpy() for k, v in out.items()})
    save.update({f"cot_{k}": v.numpy() for k, v in cots.items()})
    save.update({f"grad_{k}": v.grad.numpy() for k, v in leaf.items()})
    np.savez_compressed(os.path.join(HERE, "frosting_bg_attrs.npz"), **save)
    print({k: v.shape for k, v in save.items() if k.startswith("out_")})


if __name__ == "__main__":
    main()
