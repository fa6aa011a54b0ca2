"""Fused photometric loss of Frosting's trainers (SURVEY.md 8f2) -- host side.

`l1_dssim_loss(pred, gt, dssim_factor=0.2)` == `(1 - f) * l1_loss(pred, gt) + f * (1 - ssim(pred, gt))` of
frosting_trainers/refine.py:407-409 with frosting_utils/loss_utils.py:17-63, for [C,H,W] or [1,C,H,W] images, as one
forward kernel (+ a tiny reduction) and one backward kernel behind the C ABI (fb200_l1_dssim_forward/backward).
`torch_reference(...)` restates the reference's torch code and is the oracle used by the tests.
"""
import math

import torch
import torch.nn.functional as F

from . import _lib


class _L1DSSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, lam):
        if not pred.is_cuda:
            raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
        shape = pred.shape
        p = pred.reshape(-1, shape[-2], shape[-1]).float().contiguous()
        g = gt.reshape(-1, shape[-2], shape[-1]).to(p.device).float().contiguous()
        Cn, H, W = p.shape
        L = _lib.lib()
        dev = p.device
        maps = torch.empty((3, Cn, H, W), dtype=torch.float32, device=dev)
        partials = torch.empty((L.fb200_loss_partials(Cn, H, W),), dtype=torch.float32, device=dev)
        loss = torch.empty((1,), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.fb200_l1_dssim_forward(p.data_ptr(), g.data_ptr(), Cn, H, W, float(lam), maps.data_ptr(),
                                                partials.data_ptr(), loss.data_ptr(), _lib.stream(dev)))
        ctx.save_for_backward(p, g, maps)
        ctx.lam, ctx.shape = float(lam), shape
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g_loss):
        p, g, maps = ctx.saved_tensors
        Cn, H, W = p.shape
        dev = p.device
        gl = g_loss.reshape(1).float().contiguous()
        dpred = torch.empty_like(p)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_l1_dssim_backward(p.data_ptr(), g.data_ptr(), maps.data_ptr(), Cn, H, W, ctx.lam,
                                                          gl.data_ptr(), dpred.data_ptr(), _lib.stream(dev)))
        return dpred.reshape(ctx.shape), None, None


def l1_dssim_loss(pred: torch.Tensor, gt: torch.Tensor, dssim_factor: float = 0.2) -> torch.Tensor:
    return _L1DSSIM.apply(pred, gt, dssim_factor)


# ---- torch restatement of frosting_utils/loss_utils.py:17-63 (test oracle, also runs on CPU) --------------------
def _window(channel, dtype, device):
    g = torch.tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])   # float32, as the reference
    g = (g / g.sum()).unsqueeze(1)
    w2 = g.mm(g.t()).float().unsqueeze(0).unsqueeze(0)
    return w2.expand(channel, 1, 11, 11).contiguous().to(device=device, dtype=dtype)


def torch_reference(pred, gt, dssim_factor: float = 0.2):
    if pred.dim() == 3:
        pred, gt = pred[None], gt[None]
    ch = pred.size(-3)
    w = _window(ch, pred.dtype, pred.device)
    conv = lambda t: F.conv2d(t, w, padding=5, groups=ch)
    mu1, mu2 = conv(pred), conv(gt)
    mu1_sq, mu2_sq, mu12 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(pred * pred) - mu1_sq, conv(gt * gt) - mu2_sq, conv(pred * gt) - mu12
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim_map = ((2 * mu12 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    l1 = torch.abs(pred - gt).mean()
    return (1.0 - dssim_factor) * l1 + dssim_factor * (1.0 - ssim_map.mean())
