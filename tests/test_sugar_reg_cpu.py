"""SuGaR's SDF regulariser without a GPU: the torch restatement against golden vectors made by executing the reference's
own source (tests/golden/make_sugar_reg_golden.py), the reference's draws, the neighbour table's validation and the
exported entry points' argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, scenes, sugar

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_sugar_sdf_reg.npz")
LEAVES = ("points", "scaling", "quaternions", "strengths")


def golden():
    return np.load(GOLD)


def reference_run(z, dtype):
    """torch_reference on the golden's inputs, under torch.use_deterministic_algorithms(True) as the golden was made: the
    indexing backward's CPU scatter then sums in a fixed order."""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        leaves = {k: torch.from_numpy(z[k]).to(dtype).requires_grad_(True) for k in LEAVES}
        idx, eps = torch.from_numpy(z["idx"]), torch.from_numpy(z["eps"]).to(dtype)
        est, nrm, fields = sugar.torch_reference(*leaves.values(), torch.from_numpy(z["knn_idx"]), idx, eps,
                                                 return_fields=True)
        out = {"terms": torch.stack([est, nrm]).detach(), **{k: v.detach() for k, v in fields.items()}}
        for term, value in (("est", est), ("nrm", nrm)):
            grads = torch.autograd.grad(value, list(leaves.values()), allow_unused=True, retain_graph=True)
            for k, g in zip(LEAVES, grads):
                out[f"d{term}_d{k}"] = torch.zeros_like(leaves[k]) if g is None else g
        return out
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("tag,dtype,bar", [("f64", torch.float64, 1e-12), ("f32", torch.float32, 1e-6)])
def test_restatement_matches_reference_source(tag, dtype, bar):
    """Every tensor, every row, within `bar` of its largest golden element.  In float32 all but the normal term's
    quaternion gradient are bit-identical; that one differs by ~2e-7 because the reference's source evaluates the
    normals twice and the restatement once, so autograd sums their contributions in another order."""
    z = golden()
    out = reference_run(z, dtype)
    for k, v in out.items():
        ref = torch.from_numpy(z[f"{tag}/{k}"]).to(dtype)
        scale = float(ref.abs().max())
        err = float((v - ref).abs().max())
        assert err <= bar * max(scale, 1e-30), (k, err, scale)


def test_golden_covers_the_cases():
    z = golden()
    assert tuple(z["knn_idx"].shape) == (300, 16) and (z["knn_idx"][:, 0] == np.arange(300)).all()
    assert set(z["idx"].tolist()) <= set(np.nonzero(z["mask"])[0].tolist())
    assert {7, 8, 11} <= set(z["idx"].tolist())
    assert z["scaling"].min() < 1e-8 and (z["scaling"].min(axis=1) < 1e-6).sum() >= 2
    assert (z["f64/density"] >= 1).any() and (z["f64/density"] < 1e-3).any()
    # the normal term reaches the quaternions only; both terms reach every input except the normal term's
    for k in ("points", "scaling", "strengths"):
        assert not z[f"f64/dnrm_d{k}"].any() and np.abs(z[f"f64/dest_d{k}"]).max() > 0
    assert np.abs(z["f64/dnrm_dquaternions"]).max() > 0


def test_sampler_draws_the_reference_samples():
    z = golden()
    torch.manual_seed(int(z["seed"]))
    idx, eps = sugar.sample_in_gaussians(torch.from_numpy(z["mask"]), int(z["n_samples"]))
    assert idx.dtype == torch.int64 and eps.dtype == torch.float32
    assert torch.equal(idx, torch.from_numpy(z["idx"])) and torch.equal(eps, torch.from_numpy(z["eps"]))


def test_sampler_empty_mask_draws_nothing():
    state = torch.get_rng_state()
    idx, eps = sugar.sample_in_gaussians(torch.zeros(10, dtype=torch.bool), 1000)
    assert idx.shape == (0,) and eps.shape == (0, 3)
    assert torch.equal(state, torch.get_rng_state())


def test_quaternion_apply_is_the_unnormalised_rotation():
    g = torch.Generator().manual_seed(0)
    q, v = torch.randn(50, 4, generator=g, dtype=torch.float64), torch.randn(50, 3, generator=g, dtype=torch.float64)
    n2 = (q * q).sum(-1, keepdim=True)
    R = scenes.quaternion_to_matrix(q)
    assert torch.allclose(scenes.quaternion_apply(q, v), n2 * (R @ v[..., None])[..., 0], atol=1e-12)


def test_sugar_scene_shapes_and_table():
    sc = scenes.sugar_scene(500, 3, K=5)
    assert sc["knn_idx"].shape == (500, 5) and torch.equal(sc["knn_idx"][:, 0], torch.arange(500))
    assert sc["strengths"].shape == (500, 1) and torch.allclose(sc["quaternions"].norm(dim=-1), torch.ones(500))
    flat = sc["scaling"][:450]
    assert (flat.min(dim=-1)[0] < 0.2 * flat.max(dim=-1)[0]).float().mean() > 0.95


def test_neighbour_table_validation():
    t = sugar.SugarNeighbours(torch.tensor([[0, 1], [1, 0], [2, 1]]))
    assert t.knn_idx.dtype == torch.int32 and (t.P, t.K) == (3, 2)
    for bad in (torch.zeros(3, dtype=torch.long), torch.zeros(3, 0, dtype=torch.long),
                torch.zeros(40, 33, dtype=torch.long)):
        with pytest.raises(ValueError, match=r"\[P, K\]"):
            sugar.SugarNeighbours(bad)
    with pytest.raises(ValueError, match="integer"):
        sugar.SugarNeighbours(torch.zeros(3, 2))
    for bad in (torch.tensor([[0, 3], [1, 0], [2, 1]]), torch.tensor([[0, -1], [1, 0], [2, 1]])):
        with pytest.raises(ValueError, match=r"outside \[0, 3\)"):
            sugar.SugarNeighbours(bad)


def test_python_surface_rejects_cpu():
    sc = scenes.sugar_scene(40, 0, K=4)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        sugar.sdf_regularization(sc["points"], sc["scaling"], sc["quaternions"], sc["strengths"],
                                 sugar.SugarNeighbours(sc["knn_idx"]), torch.zeros(3, dtype=torch.long),
                                 torch.zeros(3, 3))


def test_sugar_reg_entry_points_are_exported():
    import frosting_b200 as fb
    L = _lib.lib()
    for n in ("fb200_sugar_reg_workspace_bytes", "fb200_sugar_reg_forward", "fb200_sugar_reg_backward",
              "fb200_sugar_reg_struct_size"):
        assert n in _lib.EXPORTED and hasattr(L, n)
    assert L.fb200_sugar_reg_struct_size() == C.sizeof(_lib.SugarReg)
    assert fb.sdf_regularization is sugar.sdf_regularization and fb.SugarNeighbours is sugar.SugarNeighbours
    # records + partials (two floats per block of 16 samples at K = 16, of 32 at K = 5), then with the gradient pass
    # the accumulators from the next 16-byte boundary
    P = 1 << 18
    ws = L.fb200_sugar_reg_workspace_bytes
    assert ws(P, 16, 1600, 0) == P * 80 + 2 * 4 * 100 and ws(P, 16, 1600, 1) == P * (80 + 128) + 2 * 4 * 100
    assert ws(P, 16, 1601, 0) == P * 80 + 2 * 4 * 101 and ws(P, 16, 1601, 1) == P * (80 + 128) + 816
    assert ws(P, 5, 1600, 1) == P * (80 + 128) + 2 * 4 * 50
    # below 2^18 Gaussians the accumulators are replicated R = 2^18 / P times (a power of two, at most 1024)
    assert ws(1000, 16, 1600, 1) == 1000 * (80 + 128 * 256) + 2 * 4 * 100
    assert ws(17, 16, 1600, 0) == 17 * 80 + 2 * 4 * 100
    assert ws(17, 16, 1600, 1) == 17 * (80 + 128 * 1024) + 2 * 4 * 100
    for bad in ((-1, 16, 10), (10, 0, 10), (10, 33, 10), (10, 16, -1)):
        assert ws(*bad, 1) == 0


def _reg(**kw):
    d = C.c_void_p(0x1000)
    f = dict(P=10, K=16, N=100, sampling_scale_factor=1.5)
    for n, _ in _lib.SugarReg._fields_[4:]:
        f[n] = d
    f.update(kw)
    return _lib.SugarReg(**f)


def test_sugar_reg_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    d = C.c_void_p(0x1000)
    fwd = lambda r, terms=d: L.fb200_sugar_reg_forward(C.byref(r) if r is not None else None, 1, terms, None)
    bwd = lambda r, *g: L.fb200_sugar_reg_backward(C.byref(r), *(g or (d,) * 5), None)
    err = lambda: L.fb200_last_error()
    assert fwd(None) == -1 and b"null struct" in err()
    for bad in (dict(P=-1), dict(N=-1), dict(P=0)):
        assert fwd(_reg(**bad)) == -1 and b"bad extents" in err(), bad
        assert bwd(_reg(**bad)) == -1 and b"bad extents" in err(), bad
    for K in (0, 33, -2):
        assert fwd(_reg(K=K)) == -1 and b"K must be within [1, 32]" in err()
    for n in ("d_points", "d_scaling", "d_quaternions", "d_strengths", "d_knn_idx"):
        assert fwd(_reg(**{n: None})) == -1 and b"missing Gaussian pointer" in err(), n
    for n in ("d_idx", "d_eps"):
        assert fwd(_reg(**{n: None})) == -1 and b"missing sample pointer" in err(), n
    assert fwd(_reg(d_workspace=None)) == -1 and b"missing workspace" in err()
    assert fwd(_reg(d_quaternions=C.c_void_p(0x1004))) == -1 and b"16-byte aligned" in err()
    assert fwd(_reg(d_workspace=C.c_void_p(0x1008))) == -1 and b"16-byte aligned" in err()
    assert fwd(_reg(), None) == -1 and b"missing terms output" in err()
    assert bwd(_reg(), d, d, d, None, d) == -1 and b"missing gradient pointer" in err()
    assert bwd(_reg(), None, d, d, d, d) == -1 and b"missing gradient pointer" in err()
    assert bwd(_reg(), d, d, d, C.c_void_p(0x1004), d) == -1 and b"dL/dquaternions must be 16-byte aligned" in err()
    # no Gaussians, no samples: nothing to differentiate, no launch
    assert bwd(_reg(P=0, N=0, d_points=None, d_idx=None), None, None, None, None, None) == 0
