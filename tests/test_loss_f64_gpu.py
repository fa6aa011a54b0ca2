"""Fused L1 + D-SSIM loss (csrc/loss.cu) against a float64 restatement of the same operation.

Every case computes three results from the same float32 inputs:
  ours  `l1_dssim_loss`
  R32   `loss.torch_reference` in float32 on the GPU, with cuDNN's TF32 off: the float32 arithmetic the reference's
        torch loss is written in
  R64   `loss.torch_reference` in float64, pinned to the reference's own loss_utils.py by
        tests/test_loss.py::test_float64_restatement_matches_reference_golden.  Its L1 and 1 - SSIM terms are computed
        once per image and combined in float64 for each weight and upstream gradient.

The bar is "no less accurate than the reference computing in float32", measured against float64:
  gradient  max|G - G64| <= 2 max|G32 - G64| + 1e-6 max|G64|, and the same on the 99.9th percentiles of the errors
  loss      |L - L64| <= 2 |L32 - L64| + 1e-6 |L64|
It is tight where the problem is well conditioned and honest in flat regions, where sigma^2 = E[x^2] - mu^2 cancels in
float32 for both implementations.  Two regimes have their own factor, from measurements on an H100 80GB HBM3 (700 W):
  - The loss of a half-flat image ("flat0", "flat1") is a mean of SSIM values whose float32 error is a
    cancellation residue of ~u mu^2 / C2 in the band where the flat half meets the texture, so any float32 evaluation
    order lands 1e-6..5e-5 (relative) from float64.  R32 itself, run on the image, its transpose and its mirror image,
    scatters up to 4.5e-5 (15x17, C = 3, lambda = 1), and one such run can be luckily close (45x70, C = 1, lambda =
    1: 1.6e-7 against 2.5e-6 on the transpose).  Ours reaches 2.7e-5.  Floor: 5e-5 |L64|.
  - The gradient of "flat1": inside the white half, pred == gt and every element is the rounding residue of
    c0 + 2 x c1 + y c2 with |c1|, |c2| ~ 1/C2 (below).  Ours' residue has a 99.9th percentile 2.0-2.05 times R32's at
    1080x1920 and 1200x1600 (1.2-1.4 at smaller sizes, max errors 1.1-1.6 times).  Factor 3.

pred == gt ("equal", "const"): the float64 gradient is 0 up to rounding and float32 leaves noise, so the bound is
absolute.  There the gradient is dL * lambda / N * (c0 + 2 x c1 + y c2), N = C*H*W, where c1 and c2 are window sums of
-SSIM/D and 2A/(Cc D), at most 1/C2 and 2/C2 (D >= C2 = 0.03^2), and the last two terms cancel exactly for x = y <= 1.
Rounding leaves a few u * 4/C2 (u = 2^-24), so |G - G64| <= K |dL| lambda / N with K = 64 u / C2 = 4.2e-3; each
pixel's SSIM is 1 to a few u, so |L - L64| <= 8 u lambda.  The same absolute bound holds outside the 21x21 support of a
single-pixel difference ("pixel"), where a halo or adjoint-padding error of the backward would show.

Cases: the product of 14 image sizes (1x1 to the benchmark's 1080x1920 and 1200x1600 frames, one below, at and one
above the 16x16 tile and the 11x11 window) and 7 contents; inside each, C in {1, 3, 4} times lambda in {0, 0.2, 0.5, 1}
(lambda = 1 is the SSIM gradient alone), with the layout ([C,H,W], [1,C,H,W], a non-contiguous pred view) and the
upstream gradient dL/dloss in {1, 3, -0.5, 0} cycled over them.  Each test prints its worst margins: the error as a
fraction of its bound, and in brackets the error over R32's error (for pred == gt: R32's error as a fraction of the same
bound).

Worst margins observed on the H100 (error / bound): gradient max 0.59 and 99.9th percentile 0.59 (1x1, where R32 is
exact to the last bit and the 1e-6 floor decides), 0.29 from 5x7 up for random textures, 0.99 for "flat1"'s 99.9th
percentile against factor 2 (0.66 against 3); loss 0.89 (4x4 noise); pred == gt 0.014 of K (R32: 0.15); outside a
single pixel's support 0.001 of K.  A copy of the kernel with d(SSIM)/dE[x^2] scaled by 1.001, one with the 1/N of
the gradient computed for C = 3, and one whose backward drops the last row and column of the derivative maps' halo
each fail 30 or more of the sweep's cases.
"""
import math

import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import camera_batch as cbm
from frosting_b200 import loss as fbl
from frosting_b200 import scenes
from tests.util import rel_err_stats

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (4, 4), (5, 7), (10, 11), (11, 11), (15, 17), (16, 16), (17, 16), (31, 33), (45, 70), (64, 48),
         (200, 320), (1080, 1920), (1200, 1600)]
CONTENTS = ["noise", "equal", "const", "flat1", "flat0", "over1", "pixel"]
CHANNELS = (1, 3, 4)
LAMBDAS = (0.0, 0.2, 0.5, 1.0)
UPSTREAM = (1.0, 3.0, -0.5, 0.0)
LAYOUTS = ("chw", "1chw", "strided")

FACTOR = 2.0            # ours may be at most this many times as far from float64 as R32 ...
REL_FLOOR = 1e-6        # ... plus this fraction of the float64 scale
FLAT_LOSS_FLOOR = 5e-5  # the loss of half-flat images (module docstring)
WHITE_FACTOR = 3.0      # the gradient of half-white images (module docstring)
U32 = 2.0 ** -24
C2 = 0.03 ** 2
K_DEGENERATE = 64 * U32 / C2
SUPPORT = 10            # a pixel's gradient reaches 2 * 5 pixels: two 11x11 windows


@pytest.fixture(autouse=True)
def _float32_convolutions(monkeypatch):
    """R32 must compute in float32: cuDNN would otherwise run its convolutions in TF32."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _pixel(C, H, W):
    """The single differing pixel: its support crosses the tile borders at 16 in both directions."""
    return C - 1, min(H - 1, 17), min(W - 1, 14)


def _images(content, C, H, W):
    g = torch.Generator().manual_seed(10007 * H + 101 * W + C)
    gt = torch.rand(C, H, W, generator=g)
    pred = (gt + 0.1 * torch.randn(C, H, W, generator=g)).clamp(0, 1)
    if content == "over1":                       # unclamped renders exceed 1
        pred = (2.0 * gt + 0.05 * torch.randn(C, H, W, generator=g)).clamp(0, 2)
    elif content in ("flat1", "flat0"):          # white / black backgrounds, identical in both images
        v, half = (1.0 if content == "flat1" else 0.0), (W + 1) // 2
        gt[..., :half] = v
        pred[..., :half] = v
    elif content == "equal":
        pred = gt.clone()
    elif content == "const":
        gt.fill_(0.5)
        pred = gt.clone()
    elif content == "pixel":
        pred = gt.clone()
        pred[_pixel(C, H, W)] += 0.3
    return pred, gt


def _views(pred, gt, layout):
    """(leaf, pred as the loss sees it, gt) for a layout; _chw maps the leaf's gradient back to [C,H,W]."""
    if layout == "chw":
        leaf = pred.clone().requires_grad_(True)
        return leaf, leaf, gt
    if layout == "1chw":
        leaf = pred[None].clone().requires_grad_(True)
        return leaf, leaf, gt[None]
    leaf = pred.transpose(1, 2).contiguous().requires_grad_(True)      # pred is a transposed, non-contiguous view
    return leaf, leaf.transpose(1, 2), gt


def _chw(grad, layout):
    return grad[0] if layout == "1chw" else grad.transpose(1, 2) if layout == "strided" else grad


def _eval(fn, pred, gt, lam, layout, dL):
    leaf, p, g = _views(pred, gt, layout)
    loss = fn(p, g, lam)
    assert loss.shape == ()
    (grad,) = torch.autograd.grad(loss, leaf, torch.tensor(dL, dtype=loss.dtype, device=loss.device))
    assert grad.shape == leaf.shape
    return float(loss), _chw(grad, layout).double()


def _float64_terms(pred, gt):
    """L1, its gradient, 1 - SSIM and its gradient, in float64 (torch_reference at weights 0 and 1)."""
    out = []
    for lam in (0.0, 1.0):
        p = pred.double().requires_grad_(True)
        loss = fbl.torch_reference(p, gt.double(), lam)
        (g,) = torch.autograd.grad(loss, p)
        out += [loss.item(), g]
    return out


def _ratio(a, b):
    return a / b if b > 0 else (0.0 if a == 0 else math.inf)


def _check(pred, gt, lam, layout, dL, terms, degenerate, outside=None, factor=FACTOR, loss_floor=REL_FLOOR):
    """One case; returns its margins {check: (error / bound, error / R32's error)}.  `outside`: a mask where the
    float64 gradient is 0 up to rounding (the absolute bound applies there)."""
    l1, g_l1, dssim, g_dssim = terms
    L64 = (1.0 - lam) * l1 + lam * dssim
    G64 = dL * ((1.0 - lam) * g_l1 + lam * g_dssim)
    L, G = _eval(fbl.l1_dssim_loss, pred, gt, lam, layout, dL)
    L32, G32 = _eval(fbl.torch_reference, pred, gt, lam, layout, dL)
    assert math.isfinite(L) and bool(torch.isfinite(G).all())
    e, e32 = (G - G64).abs().flatten(), (G32 - G64).abs().flatten()
    N = pred.numel()
    abs_bound = K_DEGENERATE * abs(dL) * lam / N
    m = {}
    if degenerate:
        eL, eL32 = abs(L - L64), abs(L32 - L64)
        m["grad"] = (_ratio(e.max().item(), abs_bound), _ratio(e32.max().item(), abs_bound))
        m["loss"] = (_ratio(eL, 8 * U32 * lam), _ratio(eL32, 8 * U32 * lam))
        assert e.max().item() <= abs_bound, ("grad", e.max().item(), abs_bound)
        assert eL <= 8 * U32 * lam, ("loss", L, L64)
        return m
    floor = REL_FLOOR * G64.abs().max().item()
    for name, a, b in (("grad max", e.max().item(), e32.max().item()),
                       ("grad p99.9", torch.quantile(e, 0.999).item(), torch.quantile(e32, 0.999).item())):
        m[name] = (_ratio(a, factor * b + floor), _ratio(a, b))
        assert a <= factor * b + floor, (name, a, b, floor)
    eL, eL32 = abs(L - L64), abs(L32 - L64)
    m["loss"] = (_ratio(eL, FACTOR * eL32 + loss_floor * abs(L64)), _ratio(eL, eL32))
    assert eL <= FACTOR * eL32 + loss_floor * abs(L64), ("loss", L, L32, L64)
    if outside is not None:
        eo = e[outside.flatten()].max().item()
        m["outside"] = (_ratio(eo, abs_bound), _ratio(eo, e32[outside.flatten()].max().item()))
        assert eo <= abs_bound, ("outside the support", eo, abs_bound)
    return m


def _report(capsys, tag, margins):
    worst = {}
    for m in margins:
        for k, (r, r32) in m.items():
            w = worst.setdefault(k, [0.0, 0.0])
            w[0], w[1] = max(w[0], r), max(w[1], r32)
    with capsys.disabled():
        print(f"\n[loss f64] {tag}: " + ", ".join(f"{k} {r:.3f} of bound ({r32:.3g})" for k, (r, r32) in worst.items()),
              end="")


@pytest.mark.parametrize("content", CONTENTS)
@pytest.mark.parametrize("H,W", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_fused_loss_against_float64(cuda_device, capsys, H, W, content):
    dev = cuda_device
    si = SIZES.index((H, W))
    margins = []
    for ci, C in enumerate(CHANNELS):
        pred, gt = (t.to(dev) for t in _images(content, C, H, W))
        terms = _float64_terms(pred, gt)
        outside = None
        if content == "pixel":
            c, y, x = _pixel(C, H, W)
            yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
            outside = torch.ones(C, H, W, dtype=torch.bool, device=dev)
            outside[c] = ((yy - y).abs() > SUPPORT) | ((xx - x).abs() > SUPPORT)
            if not bool(outside.any()):
                outside = None
        for li, lam in enumerate(LAMBDAS):
            layout = LAYOUTS[(si + ci + li) % len(LAYOUTS)]
            dL = UPSTREAM[(si + 2 * ci + li) % len(UPSTREAM)]
            try:
                margins.append(_check(pred, gt, lam, layout, dL, terms, content in ("equal", "const"), outside,
                                      factor=WHITE_FACTOR if content == "flat1" else FACTOR,
                                      loss_floor=FLAT_LOSS_FLOOR if content in ("flat0", "flat1") else REL_FLOOR))
            except AssertionError as ex:
                raise AssertionError(f"C={C} lambda={lam} layout={layout} dL={dL}: {ex}") from None
    _report(capsys, f"{H}x{W} {content}", margins)


@pytest.mark.parametrize("C,H,W", [(3, 45, 70), (4, 17, 16), (3, 1080, 1920)])
def test_fused_loss_gradient_is_bit_reproducible(cuda_device, C, H, W):
    """Two backwards over one forward (retain_graph) and two forwards give the same bits: the kernels reduce in a fixed
    order and the backward reads only what the forward saved."""
    dev = cuda_device
    pred, gt = (t.to(dev) for t in _images("noise", C, H, W))
    p = pred.clone().requires_grad_(True)
    up = torch.tensor(3.0, device=dev)
    l1 = fbl.l1_dssim_loss(p, gt, 0.2)
    (g1,) = torch.autograd.grad(l1, p, up, retain_graph=True)
    (g2,) = torch.autograd.grad(l1, p, up)
    l2 = fbl.l1_dssim_loss(p, gt, 0.2)
    (g3,) = torch.autograd.grad(l2, p, up)
    assert torch.equal(l1.detach().view(torch.int32), l2.detach().view(torch.int32))
    assert torch.equal(g1.view(torch.int32), g2.view(torch.int32))
    assert torch.equal(g1.view(torch.int32), g3.view(torch.int32))
    assert float(g1.abs().max()) > 0


@pytest.mark.parametrize("name,cams", [("tiny", cbm.CAMS_PER_GPU), ("c3", 1)])
def test_training_frame_with_fused_loss_matches_reference_loss(cuda_device, monkeypatch, capsys, name, cams):
    """bench.py's training frame (CameraBatch frosting / lookup / l1_dssim, its seeded ground-truth images) against the
    same frame with the loss replaced by torch_reference in float32.  Both frames render the same image, so they differ
    only by the cotangent the loss hands to the backward (shape, 1/N, upstream gradient) and the blend backward's
    atomic order: every parameter gradient within tests/util.py::rel_err_stats <= 1e-3 / 1e-3, the loss within the
    sweep's bound.  The rendered image, with its flat black background, also goes through the sweep's check."""
    dev = cuda_device
    wl = cbm.build_workload(name, dev, cams_per_gpu=cams)
    H, W = wl["H"], wl["W"]
    gtg = torch.Generator().manual_seed(99)                # as bench.py seeds rank 0's ground truth
    gts = [torch.rand(3, H, W, generator=gtg).to(dev) for _ in wl["cams"]]
    margins = []
    for i, cam in enumerate(wl["cams"]):
        rs = scenes.settings_for(cam, wl["D"], device=dev)
        runs = []
        for loss_fn in (fb.l1_dssim_loss, fbl.torch_reference):
            monkeypatch.setattr(fb, "l1_dssim_loss", loss_fn)
            step = cbm.CameraBatch(wl, dev, mode="frosting", mask="lookup", loss="l1_dssim")
            step.gt = gts
            loss = float(step.frame(i, rs, None))
            runs.append((loss, step.last["color"].detach(), {k: v.grad for k, v in step.params.items()}))
        (L, color, grads), (L32, color32, grads32) = runs
        assert torch.equal(color.view(torch.int32), color32.view(torch.int32))
        L64 = float(fbl.torch_reference(color.double(), gts[i].double(), 0.2))
        assert abs(L - L64) <= FACTOR * abs(L32 - L64) + REL_FLOOR * abs(L64), (i, L, L32, L64)
        for k in grads:
            assert float(grads32[k].abs().sum()) > 0, k
            mx, frac = rel_err_stats(grads[k], grads32[k])
            assert mx <= 1e-3 and frac <= 1e-3, (i, k, mx, frac)
        margins.append(_check(color, gts[i], 0.2, "chw", 1.0, _float64_terms(color, gts[i]), False))
    _report(capsys, f"{name} frame ({len(wl['cams'])} cameras)", margins)
