"""The float64 blend model (oracle/blend_f64.py) against the C oracle's blend (oracle/raster_oracle.c, pinned to the
reference by tests/test_oracle_golden_cpu.py), element by element, and against central differences of its own forward.

The C oracle evaluates every pair in float32 with libm's expf and recovers T by division as the reference does; its
accumulators are float64.  So |oracle - model| <= TAU_CPU * m64 + 1e-30 on every used accumulator slot (slot 3 being
half of d/d(conic.y), the oracle's dL_dconic[1]) checks the model's quirks: the straight-through 0.99 clamp, the NDC
factor, the background term, the decisions resolved from final_T.  The planted scene puts pairs within a few ulp of
1/255, where float64 and float32 can decide differently, and checks that the resolution picks the oracle's decisions
exactly (the oracle's float32 decisions are recomputed here with libm's fmaf / expf, op for op)."""
import ctypes as C
import ctypes.util
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import blend_f64, cpu
from tests.util import scene

TAU_CPU = 6e-8       # one float32 ulp; the largest ratio seen over this file is 6.3e-9


def _oracle_bwd(cam, pre, binned, fwd, dL_dpix):
    P = pre["xy"].shape[0]
    g2 = np.zeros((P, 2)); gc = np.zeros((P, 3)); go = np.zeros(P); gcol = np.zeros((P, 3))
    cpu.lib().oracle_render_bwd(
        C.c_int(P), C.c_int(cam.W), C.c_int(cam.H), cpu._p(binned["ranges"]), cpu._p(binned["point_list"]),
        cpu._p(cam.bg), cpu._p(pre["xy"]), cpu._p(pre["conic_opacity"]), cpu._p(pre["rgb"]),
        cpu._p(np.ascontiguousarray(fwd["final_T"].reshape(-1))), cpu._p(np.ascontiguousarray(fwd["n_contrib"].reshape(-1))),
        cpu._p(np.ascontiguousarray(dL_dpix, dtype=np.float32)), cpu._p(g2), cpu._p(gc), cpu._p(go), cpu._p(gcol))
    return np.concatenate([g2, gc, go[:, None], gcol], 1)      # slots 0..8


def _model(cam, pre, binned, fwd, dL_dpix, **kw):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    co = t(pre["conic_opacity"])
    return blend_f64.blend(t(pre["xy"]), co[:, :3], co[:, 3], t(pre["rgb"]), t(binned["ranges"].astype(np.int64)),
                           t(binned["point_list"].astype(np.int64)), t(fwd["n_contrib"].astype(np.int64)),
                           t(fwd["final_T"]), cam.W, cam.H, t(dL_dpix), t(cam.bg), image=t(fwd["color"]), **kw)


def _check(a_ref, r, what):
    a64, m64 = r["a64"][:, :9], r["m64"][:, :9]
    ref = torch.from_numpy(a_ref)
    bad = blend_f64.outside(ref, a64, m64, TAU_CPU)
    ex = blend_f64.excess(ref, a64, m64)
    assert not bool(bad.any()), (what, int(bad.sum()), float(ex.max()), torch.nonzero(bad)[:5].tolist())
    return float(ex.max())


CASES = [  # P, W, H, bg, seed
    (300, 61, 45, 0.7, 1),
    (1500, 97, 67, 1.0, 2),
    (3000, 131, 75, -0.4, 3),
]


@pytest.mark.parametrize("P,W,H,bgv,seed", CASES)
def test_model_matches_the_c_oracle_element_by_element(P, W, H, bgv, seed):
    cam_, g, rs = scene(P, W, H, seed, 0, "cpu", bg=bgv)
    rs = rs._replace(bg=torch.tensor([bgv, -0.5 * bgv, 0.3]))
    gen = torch.Generator().manual_seed(seed)
    op = g["opacities"].clone()
    hi = torch.rand(P, generator=gen) < 0.15
    op[hi, 0] = 0.99 + 0.01 * torch.rand(int(hi.sum()), generator=gen)          # og > 0.99: the clamp
    fwd = cpu.forward(rs, g["means3D"].numpy(), op.numpy(), shs=g["shs"][:, :1].numpy(), scales=g["scales"].numpy(),
                      rots=g["rotations"].numpy())
    cam, pre, binned = fwd["cam"], fwd["pre"], fwd["binned"]
    dp = (torch.randn(3, H, W, generator=gen) * 10 ** (3 * torch.rand(3, H, W, generator=gen) - 2)).numpy()
    dp[:, ::7] = 0.0
    ref = _oracle_bwd(cam, pre, binned, fwd, dp)
    r = _model(cam, pre, binned, fwd, dp)
    clamped = int((r["og"] > 0.99).sum())
    assert clamped >= 5, clamped
    worst = _check(ref, r, "accumulators")
    # the forward image against the oracle's float32 image
    img = torch.from_numpy(fwd["color"]).double()
    assert bool(((img - r["image64"]).abs() <= TAU_CPU * r["image_m"] + 1e-30).all())
    # pixels with no pair are the background; the undecided pairs are few and all resolved
    assert r["logT_err"] < 1e-4
    print(f"\nP={P} {W}x{H}: {r['pix'].numel()} contributing pairs, {r['undecided']} undecided resolved, "
          f"og > 0.99: {clamped}, max |oracle - model| / m64 = {worst:.2e}")


def test_model_gradient_matches_central_differences():
    """A tiny scene with every pair far from the decision thresholds and from the 0.99 clamp: the model's autograd
    (with the NDC factor and the half conic.y derivative) against central differences of its own float64 forward."""
    W, H = 19, 13
    gen = torch.Generator().manual_seed(5)
    n = 6
    xy = torch.stack([torch.rand(n, generator=gen) * (W - 1), torch.rand(n, generator=gen) * (H - 1)], 1).double()
    A = 0.05 + 0.1 * torch.rand(n, generator=gen)
    Cc = 0.05 + 0.1 * torch.rand(n, generator=gen)
    B = (torch.rand(n, generator=gen) - 0.5) * 0.8 * torch.sqrt(A * Cc)
    conic = torch.stack([A, B, Cc], 1).double()
    op = (0.3 + 0.5 * torch.rand(n, generator=gen)).double()
    col = torch.rand(n, 3, generator=gen).double()
    feat = torch.randn(n, 2, generator=gen).double()
    ranges = torch.tensor([[t * n, (t + 1) * n] for t in range(2)])
    plist = torch.arange(n).repeat(2)
    bg, xbg = torch.tensor([0.2, -0.4, 0.9]).double(), torch.tensor([0.5, -1.5]).double()
    dp, de = torch.randn(3, H, W, generator=gen).double(), torch.randn(2, H, W, generator=gen).double()

    def decisions(xy_, conic_, op_):
        """n_contrib and final_T of the float64 forward (no pixel saturates at these opacities)."""
        py, px = torch.meshgrid(torch.arange(H).double(), torch.arange(W).double(), indexing="ij")
        dx, dy = xy_[:, 0, None, None] - px, xy_[:, 1, None, None] - py
        pw = -0.5 * (conic_[:, 0, None, None] * dx * dx + conic_[:, 2, None, None] * dy * dy) - \
            conic_[:, 1, None, None] * dx * dy
        og = op_[:, None, None] * torch.exp(pw)
        ok = (og >= blend_f64.THR) & (pw <= 0)
        margin = (og / blend_f64.THR - 1).abs()
        idx = torch.arange(1, n + 1)[:, None, None].expand_as(ok)
        nc = torch.where(ok, idx, torch.zeros_like(idx)).amax(0)
        fT = torch.where(ok, 1 - og.clamp(max=0.99), torch.ones_like(og)).prod(0)
        return nc, fT, float(margin.min())

    def run(xy_, conic_, op_, col_, feat_):
        nc, fT, margin = decisions(xy_, conic_, op_)
        assert margin > 1e-3       # far from the 1/255 threshold: the decisions do not move under the perturbations
        return blend_f64.blend(xy_, conic_, op_, col_, ranges, plist, nc, fT, W, H, dp, bg, feat=feat_, ex_bg=xbg,
                               dL_dex=de)

    def loss(r):
        return float((r["image64"] * dp).sum() + (r["extra64"] * de).sum())

    r0 = run(xy, conic, op, col, feat)
    assert r0["pix"].numel() > 100
    h = 1e-6
    leaves = [(xy, 0, 0, 0.5 * W), (xy, 1, 1, 0.5 * H), (conic, 0, 2, 1.0), (conic, 1, 3, 0.5), (conic, 2, 4, 1.0),
              (op, None, 5, 1.0), (col, 0, 6, 1.0), (col, 1, 7, 1.0), (col, 2, 8, 1.0), (feat, 0, 9, 1.0),
              (feat, 1, 10, 1.0)]
    for t, c, slot, factor in leaves:
        for i in range(n):
            vals = []
            for s in (1, -1):
                args = [xy.clone(), conic.clone(), op.clone(), col.clone(), feat.clone()]
                k = [a is t for a in (xy, conic, op, col, feat)].index(True)
                if c is None:
                    args[k][i] += s * h
                else:
                    args[k][i, c] += s * h
                vals.append(loss(run(*args)))
            fd = (vals[0] - vals[1]) / (2 * h) * factor
            a = float(r0["a64"][i, slot])
            assert abs(fd - a) <= 1e-6 * max(1.0, abs(a)), (slot, i, fd, a)
    assert bool((r0["a64"][:, 11] == 0).all())


def _libm():
    return C.CDLL(ctypes.util.find_library("m"))


def test_planted_threshold_pairs_resolve_to_the_oracle_decisions():
    """Pairs within a few ulp of 1/255 (where float64 may decide otherwise than float32) and opacities past 0.99; every
    Gaussian is in every tile's list.  The model's contributing pairs must be exactly the oracle's."""
    W, H = 45, 27
    gen = torch.Generator().manual_seed(11)
    f32 = np.float32
    rows = []
    # planted: centred 1 px left of a pixel centre, op chosen so that op exp(-A / 2) sits k ulp from 1/255
    for i, k in enumerate(range(-8, 9)):
        cx, cy = 2 + 4 * (i % 10), 2 + 5 * (i // 10)
        A = 2.0 + 2.0 * float(torch.rand(1, generator=gen))
        op = blend_f64.THR * np.exp(0.5 * A) * (1 + k * 2.0 ** -24)
        rows.append((cx - 1.0, cy, A, 0.0, 3.0, op, 0.3, 0.6, 0.9))
    # opaque and clamped: op in (0.99, 1), plus mid-opacity blobs over everything
    for i in range(12):
        rows.append((float(torch.rand(1, generator=gen)) * (W - 1), float(torch.rand(1, generator=gen)) * (H - 1),
                     0.002, 0.0005, 0.003, 0.997 + 0.003 * float(torch.rand(1, generator=gen)), 0.8, 0.1, 0.4))
    for i in range(30):
        rows.append((float(torch.rand(1, generator=gen)) * (W - 1), float(torch.rand(1, generator=gen)) * (H - 1),
                     0.1, -0.02, 0.08, 0.1 + 0.4 * float(torch.rand(1, generator=gen)), 0.2, 0.9, 0.5))
    rec = np.array(rows, dtype=np.float32)
    P = rec.shape[0]
    order = torch.randperm(P, generator=gen).numpy()        # depth order: planted pairs at various list depths
    T = ((W + 15) // 16) * ((H + 15) // 16)
    pre = dict(xy=np.ascontiguousarray(rec[:, 0:2]), conic_opacity=np.ascontiguousarray(rec[:, 2:6]),
               rgb=np.ascontiguousarray(rec[:, 6:9]))
    binned = dict(ranges=np.array([[t * P, (t + 1) * P] for t in range(T)], np.uint32),
                  point_list=np.tile(order, T).astype(np.uint32))
    cam = SimpleNamespace(W=W, H=H, bg=np.array([0.25, 0.5, -0.75], np.float32))
    fwd = cpu.render_fwd(cam, pre, binned)
    dp = torch.randn(3, H, W, generator=gen).numpy()
    ref = _oracle_bwd(cam, pre, binned, fwd, dp)
    r = _model(cam, pre, binned, fwd, dp)

    # the oracle's decisions, op for op (raster_oracle.c blend_power / oracle_render_fwd)
    m = _libm()
    m.fmaf.restype = m.expf.restype = C.c_float
    m.fmaf.argtypes, m.expf.argtypes = [C.c_float] * 3, [C.c_float]
    thr = f32(1.0) / f32(255.0)
    want = set()
    nc = fwd["n_contrib"].reshape(-1)
    for p in range(W * H):
        px, py = p % W, p // W
        tile = (py // 16) * ((W + 15) // 16) + px // 16
        for pos in range(int(nc[p])):
            g = int(binned["point_list"][binned["ranges"][tile, 0] + pos])
            x, y, a, b, c, op = (f32(v) for v in rec[g, :6])
            dx, dy = f32(x + f32(-px)), f32(y + f32(-py))
            q = f32(m.fmaf(dx, f32(dx * a), f32(dy * f32(dy * c))))
            u = f32(dy * f32(dx * b))
            power = f32(m.fmaf(q, f32(-0.5), f32(-u)))
            if power > 0:
                continue
            alpha = min(f32(0.99), f32(op * f32(m.expf(power))))
            if alpha < thr:
                continue
            want.add((p, pos))
    got = set(zip(r["pix"].tolist(), r["pos"].tolist()))
    assert got == want, (len(got - want), len(want - got))
    # the planted pairs are decided by the resolution, not by float64 alone
    assert r["undecided"] >= 10, r["undecided"]
    assert int((r["og"] > 0.99).sum()) >= 20
    worst = _check(ref, r, "planted")
    print(f"\nplanted: {len(want)} contributing pairs, {r['undecided']} undecided resolved, {r['ties']} ties, "
          f"max |oracle - model| / m64 = {worst:.2e}")
