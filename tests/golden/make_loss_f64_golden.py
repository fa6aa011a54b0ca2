"""Float64 golden vectors for the photometric loss, produced by IMPORTING the reference's own
frosting_utils/loss_utils.py from a checkout of the reference project (found as oracle/build_ref.py finds it):

    python tests/golden/make_loss_f64_golden.py        # writes tests/golden/loss_f64.npz

The inputs are float32 images, as the rasterizer hands them to the loss.  The reference's `l1_loss` and `ssim` are
run on float64 copies of them: `ssim` builds its float32 window and casts it to the input's type, so this is the
reference's exact operation evaluated in float64.  Each case stores both terms and their autograd gradients w.r.t. the
prediction separately, so the test can recombine them for any weight: (1 - f) * l1 + f * (1 - ssim), f = 1 being
`ssim` alone.

Cases: C = 1, 3 and 4; images of 1x1, 5x7, 10x11 and 17x33 (below, around and above the 11x11 window and the 16x16
tiles of the CUDA kernel); a prediction above 1 as unclamped renders produce; half of the image flat white in both
images; prediction equal to the ground truth."""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.build_ref import reference_dir      # noqa: E402

SRC = os.path.join(reference_dir(), "frosting_utils", "loss_utils.py")
if not os.path.exists(SRC):
    raise SystemExit(f"{SRC} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
spec = importlib.util.spec_from_file_location("ref_loss_utils", SRC)
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

# name: (C, H, W, content)
CASES = {
    "r1x1_c1": (1, 1, 1, "noise"),
    "r5x7_c4": (4, 5, 7, "noise"),
    "r10x11_c1": (1, 10, 11, "noise"),
    "r17x33_c4": (4, 17, 33, "noise"),
    "r17x33_c3": (3, 17, 33, "noise"),
    "over1_17x33_c3": (3, 17, 33, "over1"),
    "halfwhite_24x40_c3": (3, 24, 40, "halfwhite"),
    "equal_10x11_c3": (3, 10, 11, "equal"),
}

g = torch.Generator().manual_seed(2026)
out = {}
for name, (C, H, W, content) in CASES.items():
    gt = torch.rand(1, C, H, W, generator=g)
    pred = (gt + 0.1 * torch.randn(1, C, H, W, generator=g)).clamp(0, 1)
    if content == "over1":
        pred = (2.0 * gt + 0.05 * torch.randn(1, C, H, W, generator=g)).clamp(0, 2)
    elif content == "halfwhite":
        gt[..., : W // 2] = 1.0
        pred[..., : W // 2] = 1.0
    elif content == "equal":
        pred = gt.clone()
    out[f"{name}_pred"] = pred.numpy()[0]
    out[f"{name}_gt"] = gt.numpy()[0]
    for term, fn in (("l1", ref.l1_loss), ("ssim", ref.ssim)):
        p = pred.double().requires_grad_(True)
        v = fn(p, gt.double())
        v.backward()
        out[f"{name}_{term}"] = np.float64(v.item())
        out[f"{name}_{term}_grad"] = p.grad.numpy()[0]
np.savez_compressed(os.path.join(HERE, "loss_f64.npz"), **out)
print({k: float(v) for k, v in out.items() if k.endswith(("_l1", "_ssim"))})
