"""Fused L1 + D-SSIM loss (SURVEY.md 8f2): torch restatement pinned to golden vectors made by importing the
reference's loss_utils.py (CPU test); CUDA kernels against both (GPU test)."""
import os

import numpy as np
import pytest
import torch

from frosting_b200 import loss as fbl

GOLD = os.path.join(os.path.dirname(__file__), "golden", "loss_l1dssim.npz")


def _cases():
    z = np.load(GOLD)
    for n in ("a", "b", "c"):
        yield n, torch.from_numpy(z[f"{n}_pred"]), torch.from_numpy(z[f"{n}_gt"]), float(z[f"{n}_loss"]), torch.from_numpy(z[f"{n}_grad"])


def test_torch_restatement_matches_reference_golden():
    for n, pred, gt, loss, grad in _cases():
        p = pred.clone().requires_grad_(True)
        l = fbl.torch_reference(p, gt, 0.2)
        l.backward()
        assert abs(float(l.detach()) - loss) <= 1e-7, n
        assert (p.grad - grad).abs().max().item() <= 1e-9, n


GOLD64 = os.path.join(os.path.dirname(__file__), "golden", "loss_f64.npz")


@pytest.mark.parametrize("lam", [0.0, 0.2, 0.5, 1.0])
def test_float64_restatement_matches_reference_golden(lam):
    """`torch_reference` on float64 tensors -- the oracle of tests/test_loss_f64_gpu.py -- against the reference's own
    l1_loss and ssim run in float64 (tests/golden/make_loss_f64_golden.py): C = 1, 3, 4, images from 1x1 to 17x33, a
    prediction above 1, a half-white image, prediction == ground truth.  lam = 1 is ssim alone."""
    z = np.load(GOLD64)
    names = sorted(k[: -len("_pred")] for k in z.files if k.endswith("_pred"))
    assert len(names) == 8
    for n in names:
        pred = torch.from_numpy(z[f"{n}_pred"])
        assert pred.dtype == torch.float32
        p = pred.double().requires_grad_(True)
        l = fbl.torch_reference(p, torch.from_numpy(z[f"{n}_gt"]).double(), lam)
        l.backward()
        loss = (1.0 - lam) * float(z[f"{n}_l1"]) + lam * (1.0 - float(z[f"{n}_ssim"]))
        grad = (1.0 - lam) * z[f"{n}_l1_grad"] - lam * z[f"{n}_ssim_grad"]
        assert p.grad.shape == pred.shape, n
        assert abs(float(l) - loss) <= 1e-14, (n, float(l), loss)
        # pred == gt: the gradient is 0 up to float64 rounding, so the scale is the gradient's unit 1/(C*H*W)
        err = np.abs(p.grad.numpy() - grad).max()
        assert err <= 1e-12 * max(np.abs(grad).max(), 1.0 / pred.numel()), (n, err)


def test_loss_requires_cuda():
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        fbl.l1_dssim_loss(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8))


@pytest.mark.gpu
def test_fused_loss_matches_reference(cuda_device):
    dev = cuda_device
    for n, pred, gt, loss, grad in _cases():
        p = pred.to(dev).requires_grad_(True)
        l = fbl.l1_dssim_loss(p, gt.to(dev), 0.2)
        (3.0 * l).backward()
        assert abs(float(l.detach()) - loss) <= 2e-6, (n, float(l.detach()), loss)
        err = (p.grad.cpu() / 3.0 - grad).abs().max().item()
        assert err <= 1e-3 * grad.abs().max().item() + 1e-9, (n, err, grad.abs().max().item())
    # 1080p, [1,3,H,W] input, against the torch restatement on the GPU
    g = torch.Generator().manual_seed(1)
    gt = torch.rand(1, 3, 1080, 1920, generator=g).to(dev)
    pr = (gt + 0.1 * torch.randn(1, 3, 1080, 1920, generator=g).to(dev)).clamp(0, 1)
    a = pr.clone().requires_grad_(True); b = pr.clone().requires_grad_(True)
    la = fbl.l1_dssim_loss(a, gt, 0.2); la.backward()
    lb = fbl.torch_reference(b, gt, 0.2); lb.backward()
    assert abs(float(la.detach()) - float(lb.detach())) <= 2e-6
    assert (a.grad - b.grad).abs().max().item() <= 1e-3 * b.grad.abs().max().item()
    # determinism: fixed-order reduction
    assert float(fbl.l1_dssim_loss(pr, gt, 0.2)) == float(la.detach())
