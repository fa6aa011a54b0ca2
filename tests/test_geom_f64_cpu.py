"""The float64 model of the per-Gaussian backward (oracle/geom_f64.py) pinned without a GPU: against the C oracle's
oracle_geom_bwd (itself pinned to the reference) on the same float32 accumulator records, element by element under
the per-element bound of tests/test_geom_bwd_f64_gpu.py, and against central differences of its own forward map."""
import numpy as np
import pytest
import torch

from frosting_b200 import scenes
from oracle import cpu, geom_f64
from tests.test_geom_bwd_f64_gpu import TAU
from tests.util import regime_gaussians

W, H, P = 320, 208, 4000


def _case(D, M, mod, seed):
    cam = scenes.ring_cameras(8, W, H)[3]
    rs = scenes.settings_for(cam, D, scale_modifier=mod, device="cpu")
    g = regime_gaussians(P, cam, seed, sh_coeffs=M)
    gen = torch.Generator().manual_seed(seed + 1)
    acc = (torch.randn(P, 12, generator=gen) * torch.exp(torch.randn(P, 1, generator=gen))).float()
    clamped = torch.rand(P, 3, generator=gen) < 0.3
    return cam, rs, g, acc, clamped


def _oracle(rs, g, acc, clamped, D, cov3D=None):
    """oracle_geom_bwd on every row (all rendered)."""
    c = cpu.Camera(rs)
    A = {k: np.ascontiguousarray(v.numpy(), dtype=np.float32) for k, v in g.items()}
    Pn, M = A["means3D"].shape[0], A["shs"].shape[1]
    if cov3D is None:
        cov3D = cpu.preprocess(c, A["means3D"], A["opacities"], shs=A["shs"], scales=A["scales"],
                               rots=A["rotations"])["cov3D"]
        scales, rots = A["scales"], A["rotations"]
    else:
        scales = rots = None
    a = acc.numpy()
    out = dict(means3D=np.zeros((Pn, 3), np.float32), cov3D=np.zeros((Pn, 6), np.float32),
               shs=np.zeros((Pn, M, 3), np.float32), scales=np.zeros((Pn, 3), np.float32),
               rotations=np.zeros((Pn, 4), np.float32))
    p = cpu._p
    cpu.lib().oracle_geom_bwd(
        cpu.C.c_int(Pn), cpu.C.c_int(c.D), cpu.C.c_int(M), p(A["means3D"]), p(np.ones(Pn, np.int32)), p(A["shs"]),
        p(np.ascontiguousarray(clamped.numpy(), dtype=np.uint8)), p(scales), p(rots), cpu.C.c_float(c.mod),
        p(np.ascontiguousarray(cov3D, dtype=np.float32)), p(c.view), p(c.proj), p(c.campos), cpu.C.c_int(c.W),
        cpu.C.c_int(c.H), cpu.C.c_float(c.tanx), cpu.C.c_float(c.tany), p(np.ascontiguousarray(a[:, 0:2])),
        p(np.ascontiguousarray(a[:, 2:5])), p(np.ascontiguousarray(a[:, 6:9])), p(out["means3D"]), p(out["cov3D"]),
        p(out["shs"]), p(out["scales"]), p(out["rotations"]))
    return {k: torch.from_numpy(v) for k, v in out.items()}


def _guard_decided(cam, means):
    """Rows whose float32 and float64 guard-band decisions cannot differ."""
    rx, ry = geom_f64.guard_ratio(cam, means)
    return ((rx - 1).abs() > 1e-6) & ((ry - 1).abs() > 1e-6)


def _compare(name, o32, g64, m64, keep):
    r = geom_f64.excess(o32[keep], g64[keep], m64[keep])
    bad = geom_f64.outside(o32[keep], g64[keep], m64[keep], TAU)
    assert not bool(bad.any()), (name, int(bad.sum()), float(r.max()))
    return float(r.max())


@pytest.mark.parametrize("D,M,mod", [(0, 1, 0.6), (1, 9, 1.0), (2, 9, 1.7), (3, 16, 0.6), (3, 20, 1.7)])
def test_model_matches_the_c_oracle_on_every_element(D, M, mod):
    cam, rs, g, acc, clamped = _case(D, M, mod, 100 + 7 * D + M)
    cam64 = geom_f64.Camera(rs)
    keep = _guard_decided(cam64, g["means3D"])
    assert float(keep.double().mean()) > 0.999
    # the regimes are there: guard band crossed, raw quaternion norms far from 1
    rx, ry = geom_f64.guard_ratio(cam64, g["means3D"])
    assert float((rx > 1).double().mean()) > 0.1 and float((ry > 1).double().mean()) > 0.1
    qn = g["rotations"].norm(dim=1)
    assert float(((qn < 0.5) | (qn > 2)).double().mean()) > 0.2
    ref = _oracle(rs, g, acc, clamped, D)
    g64, m64 = geom_f64.splat_grads(cam64, acc.double(), clamped=clamped, D=D, means3D=g["means3D"],
                                    opacities=g["opacities"], scales=g["scales"], rotations=g["rotations"], shs=g["shs"])
    worst = {}
    for k in ("means3D", "scales", "rotations", "shs"):
        worst[k] = _compare(k, ref[k], g64[k], m64[k], keep)
    assert float(ref["shs"][:, (D + 1) ** 2:].abs().sum()) == 0.0
    print(D, M, mod, worst)


def test_model_matches_the_c_oracle_with_a_precomputed_covariance():
    D, M = 2, 9
    cam, rs, g, acc, clamped = _case(D, M, 1.0, 5)
    cam64 = geom_f64.Camera(rs)
    R = geom_f64.rotation_rows(g["rotations"].double())
    S = R.transpose(-1, -2) @ (R * (g["scales"].double() ** 2)[:, :, None])
    cov3D = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].float()
    keep = _guard_decided(cam64, g["means3D"])
    ref = _oracle(rs, g, acc, clamped, D, cov3D=cov3D.numpy())
    g64, m64 = geom_f64.splat_grads(cam64, acc.double(), clamped=clamped, D=D, means3D=g["means3D"],
                                    opacities=g["opacities"], cov3D=cov3D, shs=g["shs"])
    for k in ("means3D", "cov3D", "shs"):
        _compare(k, ref[k], g64[k], m64[k], keep)


def test_model_backward_is_the_derivative_of_its_forward_map():
    """Central differences of L = sum_k out_k acc_k at rows away from the guard band and the colour clamp, scale
    modifier 1 (d(scale) then is the true derivative); the conic's det^2 / (det^2 + 1e-7) factor is below the
    tolerance."""
    D, M = 3, 16
    cam, rs, g, acc, _ = _case(D, M, 1.0, 9)
    cam64 = geom_f64.Camera(rs)
    rx, ry = geom_f64.guard_ratio(cam64, g["means3D"])
    unclamped = torch.zeros(P, 3, dtype=torch.bool)
    col = geom_f64.splat_map(cam64, g["means3D"].double(), g["opacities"].double(), scales=g["scales"].double(),
                             rotations=g["rotations"].double(), shs=g["shs"].double(), D=D, clamped=unclamped)[:, 6:]
    # inside the guard band, colours clear of the clamp: the map is smooth there
    rows = torch.nonzero((rx < 0.9) & (ry < 0.9) & (col > 0.05).all(1)).flatten()[:12]
    assert len(rows) == 12
    x = {k: v[rows].double() for k, v in g.items()}
    a = acc[rows].double()
    clamped = unclamped[rows]

    def loss(x):
        out = geom_f64.splat_map(cam64, x["means3D"], x["opacities"], scales=x["scales"], rotations=x["rotations"],
                                 shs=x["shs"], D=D, clamped=clamped)
        return (out * a[:, :geom_f64.N_SLOTS]).sum(1)

    g64, m64 = geom_f64.splat_grads(cam64, a, clamped=clamped, D=D, **x)
    for k in ("means3D", "scales", "rotations", "shs", "opacities"):
        flat = x[k].reshape(len(rows), -1)
        for j in range(flat.shape[1]):
            h = 1e-6 * flat[:, j].abs().clamp_min(1e-3)
            up, dn = {**x}, {**x}
            up[k] = (flat + torch.nn.functional.one_hot(torch.tensor(j), flat.shape[1]) * h[:, None]).view_as(x[k])
            dn[k] = (flat - torch.nn.functional.one_hot(torch.tensor(j), flat.shape[1]) * h[:, None]).view_as(x[k])
            fd = (loss(up) - loss(dn)) / (2 * h)
            mine = g64[k].reshape(len(rows), -1)[:, j]
            mag = m64[k].reshape(len(rows), -1)[:, j]
            assert bool(((fd - mine).abs() <= 1e-4 * mag + 1e-9).all()), (k, j, fd, mine)
