"""SuGaR's SDF regulariser of the coarse stage (SURVEY.md row a23) -- host side of csrc/sugar_reg.cu.

From iteration 9 000 on, Frosting's coarse trainers (`-r dn_consistency`, `-r density`) add two losses every step
(frosting_trainers/coarse_density_and_dn_consistency.py:735-833): a million points drawn inside the Gaussians rendered
this step, SuGaR's density field at each from its owner's tracked neighbours, the density-mode SDF-estimation loss and
the "better normal" loss.  Here:

    neighbours = SugarNeighbours(sugar.knn_idx)                   # after each reset_neighbors (every 500 steps)
    idx, eps = sample_in_gaussians(radii > 0, 1_000_000)           # the reference's own draws
    est, nrm = sdf_regularization(sugar.points, sugar.scaling, sugar.quaternions, sugar.strengths, neighbours, idx, eps)
    loss = loss + 0.2 * est + 0.2 * nrm

`sdf_regularization` is one autograd.Function: one forward call (three kernels and a memset) that also differentiates
both terms, and one backward kernel over the Gaussians.  `torch_reference` restates the reference's lines in torch for
any dtype; it is the tests' oracle.
"""
import ctypes as C

import torch

from . import _lib, scenes
from ._lib import ptr, stream

MAX_K = 32


class SugarNeighbours:
    """The tracked-neighbour table knn_idx [P,K] (reset_neighbors, sugar_model.py:1044-1061; K = 16 in the trainers,
    self included), validated once -- shape, 1 <= K <= 32, every index in [0, P) -- and kept as int32 on its device."""

    def __init__(self, knn_idx):
        if knn_idx.dim() != 2 or not 1 <= knn_idx.shape[1] <= MAX_K:
            raise ValueError(f"knn_idx must be [P, K] with 1 <= K <= {MAX_K}, got {tuple(knn_idx.shape)}")
        if knn_idx.dtype.is_floating_point or knn_idx.dtype == torch.bool:
            raise ValueError(f"knn_idx must hold integer indices, got {knn_idx.dtype}")
        self.P, self.K = int(knn_idx.shape[0]), int(knn_idx.shape[1])
        if self.P > 0 and (int(knn_idx.min()) < 0 or int(knn_idx.max()) >= self.P):
            raise ValueError(f"knn_idx holds an index outside [0, {self.P})")
        self.knn_idx = knn_idx.to(torch.int32).contiguous()


def sample_in_gaussians(mask, n_samples):
    """(idx [N] int64, eps [N,3] float32): the draws of sample_points_in_gaussians (sugar_model.py:916-959) with
    probabilities_proportional_to_volume=False, by the same torch calls in the same order -- `multinomial` over the
    masked Gaussians, then `randn_like` of the [N,3] points -- so a seeded generator gives the reference's samples,
    on any device.  The masked count is read back to the host, as the reference does.  An empty mask draws nothing and
    gives N = 0 (the reference skips the terms then)."""
    mask = mask.reshape(-1).bool()
    dev = mask.device
    valid = torch.arange(mask.numel(), device=dev)[mask]
    if valid.numel() == 0:
        return valid, torch.zeros(0, 3, device=dev)
    areas = torch.ones(valid.numel(), device=dev).abs()
    probs = areas / areas.sum(dim=-1, keepdim=True)
    idx = valid[torch.multinomial(probs, num_samples=n_samples, replacement=True)]
    eps = torch.randn(idx.numel(), 3, device=dev)
    return idx, eps


def _operand(t, name, shape, dev):
    if t.device != dev or t.dtype != torch.float32 or tuple(t.shape) != shape:
        raise ValueError(f"{name} must be a float32 {list(shape)} tensor on {dev}, got {t.dtype} "
                         f"{list(t.shape)} on {t.device}")
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


class _SdfRegularization(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, scaling, quaternions, strengths, knn, idx, eps, f, grad):
        P, K, N = knn.shape[0], knn.shape[1], idx.numel()
        dev = points.device
        ctx.shapes = [t.shape for t in (points, scaling, quaternions, strengths)]
        ctx.empty = N == 0
        if ctx.empty:
            return points.new_zeros(()), points.new_zeros(())
        L = _lib.lib()
        ws = torch.empty(L.fb200_sugar_reg_workspace_bytes(P, K, N, int(grad)), dtype=torch.uint8, device=dev)
        ops = (points, scaling, quaternions, strengths.reshape(P), knn, idx, eps)
        st = _lib.SugarReg(P=P, K=K, N=N, sampling_scale_factor=float(f),
                           **{n: ptr(t) for n, t in zip(("d_points", "d_scaling", "d_quaternions", "d_strengths",
                                                         "d_knn_idx", "d_idx", "d_eps"), ops)},
                           d_workspace=ptr(ws))
        terms = torch.empty(2, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.fb200_sugar_reg_forward(C.byref(st), int(grad), ptr(terms), stream(dev)))
        if grad:
            ctx.st, ctx.keep = st, ops + (ws,)      # the struct points into these until the backward
        return terms[0], terms[1]

    @staticmethod
    def backward(ctx, g_est, g_nrm):
        grads = [torch.zeros(s, dtype=torch.float32, device=g_est.device) if ctx.empty else None for s in ctx.shapes]
        if not ctx.empty:
            dev = g_est.device
            up = torch.stack([g_est.reshape(()), g_nrm.reshape(())]).float().contiguous()
            grads = [torch.empty(s, dtype=torch.float32, device=dev) for s in ctx.shapes]
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().fb200_sugar_reg_backward(C.byref(ctx.st), ptr(up), *[ptr(g) for g in grads],
                                                               stream(dev)))
        return (*grads, None, None, None, None, None)


def sdf_regularization(points, scaling, quaternions, strengths, neighbours, idx, eps, sampling_scale_factor=1.5):
    """(estimation term, normal term) of SuGaR's SDF regulariser, unweighted, differentiable with respect to points
    [P,3], scaling [P,3], quaternions [P,4] and strengths [P,1] -- the activated tensors the trainer hands the
    rasterizer, float32 CUDA.  `neighbours` is a SugarNeighbours over the same P; `idx` [N] (in [0, P)) and `eps` [N,3]
    come from `sample_in_gaussians`.  N = 0 gives two zeros and zero gradients without a launch.  A sample whose owner
    lies outside [0, P) is skipped by the kernels and makes both terms NaN (checked on the device: no host read-back).
    The gradient pass runs only when autograd will need it: grad mode on and an input that requires grad."""
    if not points.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    dev = points.device
    P = points.shape[0]
    if neighbours.P != P or neighbours.knn_idx.device != dev:
        raise ValueError(f"neighbours cover {neighbours.P} Gaussians on {neighbours.knn_idx.device}, the scene {P} on {dev}")
    args = [_operand(t, n, s, dev) for t, n, s in ((points, "points", (P, 3)), (scaling, "scaling", (P, 3)),
                                                   (quaternions, "quaternions", (P, 4)),
                                                   (strengths, "strengths", tuple(strengths.shape)))]
    if strengths.numel() != P:
        raise ValueError(f"strengths must hold one value per Gaussian ([P,1]), got {list(strengths.shape)}")
    if idx.dim() != 1 or idx.device != dev or idx.dtype != torch.int64:
        raise ValueError("idx must be an int64 [N] tensor on the scene's device")
    N = idx.numel()
    eps = _operand(eps, "eps", (N, 3), dev)
    if N >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 samples")
    # decided here: inside Function.forward grad mode is off and needs_input_grad ignores torch.no_grad()
    grad = torch.is_grad_enabled() and any(t.requires_grad for t in (points, scaling, quaternions, strengths))
    return _SdfRegularization.apply(*args, neighbours.knn_idx, idx.contiguous(), eps, float(sampling_scale_factor),
                                    grad)


def torch_reference(points, scaling, quaternions, strengths, knn_idx, idx, eps, sampling_scale_factor=1.5,
                    return_fields=False):
    """The reference's own lines in torch, for any dtype and device: sample_points_in_gaussians' sample (:955-957),
    get_covariance(return_sqrt, inverse_scales) (:755-761), get_field_values (:1296-1312) with get_beta 'average'
    (:1226), get_smallest_axis (:970-975) and the trainer's density-mode estimation and better-normal losses
    (coarse_density_and_dn_consistency.py:758-794, 808-833).  With `return_fields`, also the per-sample density d,
    beta and target t."""
    x = points[idx] + scenes.quaternion_apply(quaternions[idx], sampling_scale_factor * scaling[idx] * eps)
    inv_scaled_rotation = scenes.quaternion_to_matrix(quaternions) * (1. / scaling.clamp(min=1e-8))[:, None]
    closest = knn_idx[idx]
    shift = x[:, None] - points[closest]
    warped = inv_scaled_rotation[closest].transpose(-1, -2) @ shift[..., None]
    opacities = (warped[..., 0] * warped[..., 0]).sum(dim=-1).clamp(min=0., max=1e8)
    opacities = strengths[closest][..., 0] * torch.exp(-1. / 2 * opacities)
    density = opacities.sum(dim=-1)
    beta = scaling.min(dim=-1)[0][closest].mean(dim=1)
    rotations = scenes.quaternion_to_matrix(quaternions)
    axis = scaling.min(dim=-1)[1][..., None, None].expand(-1, 3, -1)
    normals = rotations.gather(2, axis).squeeze(dim=2)
    own = normals[idx]
    sdf = ((x - points[idx]) * own).sum(dim=-1)
    target = torch.exp(-0.5 * sdf.pow(2) / beta.pow(2))
    estimation = (density - target).abs().mean()
    closest_min_scaling = scaling.min(dim=-1)[0][closest].detach().view(len(x), -1)
    m = normals[closest]
    m = m * torch.sign((m * own[:, None]).sum(dim=-1, keepdim=True)).detach()
    w = ((x[:, None] - points[closest]) * m).sum(dim=-1).abs().detach()
    w = opacities.detach() * w / closest_min_scaling.clamp(min=1e-6) ** 2
    w = w / w.sum(dim=-1).detach().unsqueeze(-1).clamp(min=1e-6)
    normal = (own - (w[..., None] * m).sum(dim=-2)).pow(2).sum(dim=-1).mean()
    if return_fields:
        return estimation, normal, dict(density=density, beta=beta, target=target)
    return estimation, normal
