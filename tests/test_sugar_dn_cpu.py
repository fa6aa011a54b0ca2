"""SuGaR's depth-normal consistency without a GPU: the torch restatements against golden vectors made by executing the
reference's own source (tests/golden/make_sugar_dn_golden.py), the Python surface's argument checks and the exported
entry points' argument errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, scenes, sugar_dn

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_sugar_dn.npz")
LEAVES = ("points", "scaling", "quaternions")
IMAGES = ("1x1", "2x5", "3x3", "23x37", "40x64", "23x37_perm")


def golden():
    return np.load(GOLD)


def feature_run(z, dtype):
    leaves = {k: torch.from_numpy(z[k]).to(dtype).requires_grad_(True) for k in LEAVES}
    view = torch.from_numpy(z["cam_perm/w2c"]).T.to(dtype)
    feats = sugar_dn.torch_reference_features(*leaves.values(), view, torch.from_numpy(z["cam_perm/campos"]).to(dtype))
    grads = torch.autograd.grad(feats, list(leaves.values()), grad_outputs=torch.from_numpy(z["cot"]).to(dtype),
                                allow_unused=True)
    out = {"features": feats.detach()}
    for k, g in zip(LEAVES, grads):
        out[f"dfeatures_d{k}"] = torch.zeros_like(leaves[k]) if g is None else g
    return out


def loss_run(z, name, dtype):
    dn = torch.from_numpy(z[f"img_{name}/dn"]).to(dtype).requires_grad_(True)
    loss = sugar_dn.torch_reference_loss(dn, torch.from_numpy(z[f"img_{name}/view"]).to(dtype),
                                         torch.from_numpy(z[f"img_{name}/proj"]).to(dtype))
    (g,) = torch.autograd.grad(loss, [dn], allow_unused=True)
    return {f"loss_{name}": loss.detach(), f"dloss_ddn_{name}": torch.zeros_like(dn) if g is None else g}


@pytest.mark.parametrize("tag,dtype,bar", [("f64", torch.float64, 1e-12), ("f32", torch.float32, 1e-6)])
def test_restatement_matches_reference_source(tag, dtype, bar):
    """Every tensor within `bar` of its largest golden element (a scalar: of itself)."""
    z = golden()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = feature_run(z, dtype)
        for name in IMAGES:
            out.update(loss_run(z, name, dtype))
    finally:
        torch.use_deterministic_algorithms(prev)
    for k, v in out.items():
        ref = torch.from_numpy(np.asarray(z[f"{tag}/{k}"])).to(dtype)
        scale = float(ref.abs().max())
        err = float((v - ref).abs().max())
        assert err <= bar * max(scale, 1e-30), (k, err, scale)


def test_golden_covers_the_cases():
    z = golden()
    s, f = z["scaling"], z["f64/features"]
    assert (s[3, 0] == s[3, 1] < s[3, 2]) and (s[4] == s[4, 0]).all()
    assert f[6, 1] == 0.0 and f[6, 2] == 0.0                     # sign 0: a zero normal
    assert not z["f64/dfeatures_dscaling"].any() and np.abs(z["f64/dfeatures_dquaternions"][6]).max() == 0.0
    assert np.abs(z["f64/dfeatures_dquaternions"]).max() > 0 and np.abs(z["f64/dfeatures_dpoints"]).max() > 0
    for name in ("1x1", "2x5"):
        assert z[f"f64/loss_{name}"] == 1.0 and not z[f"f64/dloss_ddn_{name}"].any()
    dn = z["img_23x37/dn"]
    assert (dn[0] == 0).any() and ((dn[1] ** 2 + dn[2] ** 2) > 1).any()
    # past the clamp the normal channels' gradient is the -dn[1:] part alone; on a border pixel that is zero
    over = (dn[1] ** 2 + dn[2] ** 2) > 1
    over[1:-1, 1:-1] = False
    assert over.any() and not z["f64/dloss_ddn_23x37"][1:, over].any()
    # background pixels inside the image reach the normalize's eps branch: gradients of 1e12 scale
    assert np.abs(z["f64/dloss_ddn_23x37"][0]).max() > 1e6


def test_python_surface_checks_arguments():
    sc = scenes.sugar_scene(40, 0, K=1)
    cam = scenes.make_camera(32, 24)
    rs = scenes.settings_for(cam, 0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        sugar_dn.depth_normal_features(sc["points"], sc["scaling"], sc["quaternions"], rs)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        sugar_dn.depth_normal_consistency(torch.zeros(3, 24, 32), rs)
    meta = torch.device("meta")
    for bad in (torch.zeros(40, 3, dtype=torch.float64, device=meta), torch.zeros(40, 4, device=meta)):
        with pytest.raises(ValueError, match="points must be a float32"):
            sugar_dn._operand(bad, "points", (40, 3), meta)


def test_dn_entry_points_are_bound_and_exported():
    import frosting_b200 as fb
    L = _lib.lib()
    for n in ("fb200_sugar_dn_features", "fb200_sugar_dn_features_backward", "fb200_sugar_dn_partials",
              "fb200_sugar_dn_loss_forward", "fb200_sugar_dn_loss_backward"):
        assert n in _lib.EXPORTED and hasattr(L, n)
    assert fb.depth_normal_features is sugar_dn.depth_normal_features
    assert fb.depth_normal_consistency is sugar_dn.depth_normal_consistency
    # one partial per 16 x 16 tile; 0 for an empty image
    assert L.fb200_sugar_dn_partials(1080, 1920) == 68 * 120 and L.fb200_sugar_dn_partials(17, 33) == 2 * 3
    assert L.fb200_sugar_dn_partials(0, 10) == 0 and L.fb200_sugar_dn_partials(10, -1) == 0


def test_dn_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    d = C.c_void_p(0x1000)
    err = lambda: L.fb200_last_error()
    feat = lambda P=10, *p: L.fb200_sugar_dn_features(P, *(p or (d,) * 6), None)
    assert feat(-1) == -1 and b"P must be >= 0" in err()
    for i in range(5):
        args = [d] * 6
        args[i] = None
        assert feat(10, *args) == -1 and b"missing input pointer" in err(), i
    assert feat(10, d, d, C.c_void_p(0x1004), d, d, d) == -1 and b"16-byte aligned" in err()
    assert feat(10, d, d, d, d, d, None) == -1 and b"missing features output" in err()
    assert L.fb200_sugar_dn_features(0, None, None, None, None, None, None, None) == 0
    fbwd = lambda *p: L.fb200_sugar_dn_features_backward(10, *p, None)
    for i in range(6, 9):
        args = [d] * 8
        args[i - 1] = None
        assert fbwd(*args) == -1 and b"missing gradient pointer" in err(), i
    assert fbwd(*([d] * 7 + [C.c_void_p(0x1008)])) == -1 and b"dL/dquaternions must be 16-byte aligned" in err()
    fwd = lambda H=8, W=8, *p: L.fb200_sugar_dn_loss_forward(d, H, W, *(p or (d,) * 4), None)
    for H, W in ((0, 8), (8, 0), (-1, 3)):
        assert fwd(H, W) == -1 and b"bad image size" in err()
    assert L.fb200_sugar_dn_loss_forward(None, 8, 8, d, d, d, d, None) == -1 and b"missing input pointer" in err()
    assert fwd(8, 8, None, d, d, d) == -1 and b"missing input pointer" in err()
    assert fwd(8, 8, d, d, None, d) == -1 and b"missing output pointer" in err()
    assert fwd(8, 8, d, d, d, None) == -1 and b"missing output pointer" in err()
    bwd = lambda *p: L.fb200_sugar_dn_loss_backward(d, 8, 8, d, d, *p, None)
    assert bwd(None, d) == -1 and b"missing gradient pointer" in err()
    assert bwd(d, None) == -1 and b"missing gradient pointer" in err()
