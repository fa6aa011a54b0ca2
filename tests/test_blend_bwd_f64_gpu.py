"""The blend backward (csrc/render_bwd.cu) element by element against its float64 model (oracle/blend_f64.py).

The forward and backward run through the C ABI; the test reads back what the blend backward consumed -- the
per-Gaussian records (fb200_layout.geom_rec), ranges, point list, n_contrib, final_T and the forward's hit lists
(img_last_entry, bin_sub_hits) -- and the accumulator record it wrote (geom_acc).  The model resolves the forward's
decisions from final_T and differentiates the float64 blend.  Every used slot of every Gaussian must satisfy

    |a32 - a64| <= TAU * m64 + 1e-30,

no fraction allowance and no excluded rows; rows that were not rendered or have no contributing pair are exactly 0,
slots beyond the extra channel count are exactly 0, and dL/dfeatures is the record's slots 9.. bit for bit.  The colour
and extra images are within TAU_IMG of the float64 forward, per pixel.  The geometry buffer is NaN-poisoned before the
forward; the first backward relies on the forward's accumulator clear (acc_zeroed_by_forward = 1), a second backward
over the same forward clears them itself (= 0) and must give the same record, not twice it.

What the forward hands the backward is pinned too: for every pixel the first last_entry[p] entries of its sub-tile's hit
list are Gaussians of the tile list in strictly increasing list position, they include every pair the model resolved
as contributing, and the last of them is the pixel's last contributor.  From those lists and the resolved decisions the
test recomputes which paths the kernel's 16-entry blocks take (phase 1 full / with skipped slots, phase 2 dense /
sparse, phase 3 full / partial, tail blocks, sub-tiles with nothing to do) and asserts each ran in every case, along
with minimum shares of the regimes the scenes are built for (tests/util.blend_regime_gaussians).

TAU is more than ten times the largest |a32 - a64| / m64 observed on an H100 (sm_90a build) over these cases,
OBSERVED."""
import ctypes as C

import pytest
import torch

from frosting_b200 import _lib, scenes
from frosting_b200._lib import Extra, Grads, Inputs, Params, Workspace
from oracle import blend_f64
from tests.util import blend_regime_gaussians

pytestmark = pytest.mark.gpu

OBSERVED = 7.2e-9      # largest |a32 - a64| / m64 on an H100 80GB HBM3 (700 W) over every case of this file: dL/dg, ch=2
TAU = 1e-7
OBSERVED_IMG = 3.8e-8  # largest |image32 - image64| / image_m, same runs
TAU_IMG = 4e-7
W, H = 330, 203              # not multiples of 8, 4 or 16; W != H
BG = (0.3, -0.6, 1.2)
EX_BG = (0.7, -1.3, 0.25)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _run(cam, g, ch, seed, dev):
    """Forward with a NaN-poisoned geometry buffer and acc_zeroed_by_forward = 1, backward, then a second backward
    with acc_zeroed_by_forward = 0; returns everything the test reads back."""
    L = _lib.lib()
    P = g["means3D"].shape[0]
    gen = torch.Generator().manual_seed(seed)
    # cotangents over six decades, exactly zero on a tenth of the pixels
    cot = lambda c: (torch.randn(c, H, W, generator=gen) * 10 ** torch.empty(c, H, W).uniform_(-4, 2, generator=gen)
                     * (torch.rand(1, H, W, generator=gen) > 0.1)).to(dev)
    dpix = cot(3)
    ex = dict(ch=ch)
    if ch:
        ex.update(feat=torch.randn(P, ch, generator=gen).to(dev), bg=torch.tensor(EX_BG[:ch], device=dev),
                  out=torch.full((ch, H, W), float("nan"), device=dev), dout=cot(ch),
                  dfeat=torch.full((P, ch), float("nan"), device=dev))
        extra = Extra(channels=ch, d_features=_p(ex["feat"]), d_background=_p(ex["bg"]), d_out=_p(ex["out"]),
                      d_dL_dout=_p(ex["dout"]), d_dL_dfeatures=_p(ex["dfeat"]))
    rs = scenes.settings_for(cam, 0, bg=torch.tensor(BG), device=dev)
    prm = Params(P=P, sh_degree=0, sh_coeffs=0, image_width=W, image_height=H, tanfovx=float(rs.tanfovx),
                 tanfovy=float(rs.tanfovy), scale_modifier=1.0, prefiltered=0, debug=0,
                 extra=C.addressof(extra) if ch else None)
    t = dict(bg=rs.bg.contiguous(), view=rs.viewmatrix.contiguous(), proj=rs.projmatrix.contiguous(),
             campos=rs.campos.contiguous())
    inp = Inputs(d_background=_p(t["bg"]), d_means3D=_p(g["means3D"]), d_colors_precomp=_p(g["colors"]),
                 d_opacities=_p(g["opacities"]), d_scales=_p(g["scales"]), d_rotations=_p(g["rotations"]),
                 d_viewmatrix=_p(t["view"]), d_projmatrix=_p(t["proj"]), d_campos=_p(t["campos"]))
    geom = torch.full((L.fb200_geom_bytes(P),), 255, dtype=torch.uint8, device=dev)     # NaN in every float
    image = torch.empty(L.fb200_image_bytes(W, H), dtype=torch.uint8, device=dev)
    status = torch.zeros(_lib.FB200_STATUS_WORDS, dtype=torch.int32, device=dev)
    ws = Workspace(d_geom=geom.data_ptr(), geom_bytes=geom.numel(), d_image=image.data_ptr(), image_bytes=image.numel(),
                   d_binning=None, binning_bytes=0, binning_capacity=0, d_status=status.data_ptr(),
                   acc_zeroed_by_forward=1, h_status=None)
    color = torch.empty(3, H, W, device=dev)
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(L.fb200_forward_geometry(C.byref(prm), C.byref(inp), C.byref(ws), _p(radii), stream))
    R = max(int(status[_lib.ST_NUM_RENDERED]), 1)
    binning = torch.empty(L.fb200_binning_bytes(R), dtype=torch.uint8, device=dev)
    ws.d_binning, ws.binning_bytes, ws.binning_capacity = binning.data_ptr(), binning.numel(), R
    _lib.check(L.fb200_forward_raster(C.byref(prm), C.byref(inp), C.byref(ws), _p(color), _p(radii), stream))
    nan = lambda *s: torch.full(s, float("nan"), device=dev)
    out = dict(means2D=nan(P, 3), colors=nan(P, 3), opacities=nan(P, 1), means3D=nan(P, 3), scales=nan(P, 3),
               rotations=nan(P, 4))
    grads = Grads(d_dL_dmeans2D=_p(out["means2D"]), d_dL_dcolors=_p(out["colors"]), d_dL_dopacity=_p(out["opacities"]),
                  d_dL_dmeans3D=_p(out["means3D"]), d_dL_dscales=_p(out["scales"]),
                  d_dL_drotations=_p(out["rotations"]), sparse_rows=0)
    v = _lib.workspace_views(geom, image, binning, P, W, H, R, R)
    accs, dfeats = [], []
    for zeroed in (1, 0):
        ws.acc_zeroed_by_forward = zeroed
        _lib.check(L.fb200_backward(C.byref(prm), C.byref(inp), C.byref(ws), _p(radii), _p(dpix), C.byref(grads),
                                    stream))
        torch.cuda.synchronize(dev)
        accs.append(v["acc"].clone())
        if ch:
            dfeats.append(ex["dfeat"].clone())
    assert int(status[_lib.ST_OVERFLOW]) == 0
    return dict(P=P, R=R, radii=radii, accs=accs, dfeats=dfeats, color=color, dpix=dpix, ex=ex,
                rec=v["rec"].clone(), final_T=v["final_T"].flatten().clone(), n_contrib=v["n_contrib"].flatten().long(),
                last_entry=v["last_entry"].flatten().long(), ranges=v["ranges"].long(),
                point_list=v["point_list"].long(), sub_hits=v["sub_hits"].long())


def _subtiles(dev):
    """Per pixel (row-major): sub-tile id (8 per tile, w = 2 * row + col) and lane (8 x 4, row-major)."""
    py, px = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    px, py = px.reshape(-1), py.reshape(-1)
    tile = (py // 16) * ((W + 15) // 16) + px // 16
    w = ((py % 16) // 4) * 2 + (px % 16) // 8
    lane = (py % 4) * 8 + px % 8
    return tile * 8 + w, lane


def _hit_lists_and_paths(f, m, dev):
    """Pins the hit lists against the resolved decisions and returns the kernel-path counts."""
    T = f["ranges"].shape[0]
    start, end = f["ranges"][:, 0], f["ranges"][:, 1]
    n_t = end - start
    sid, lane = _subtiles(dev)
    le = f["last_entry"]
    NS = 8 * T
    top = torch.zeros(NS, dtype=torch.int64, device=dev).scatter_reduce(0, sid, le, "amax")
    # every entry below a sub-tile's top: sub-tile, entry number, Gaussian, position in the tile list
    s_e = torch.repeat_interleave(torch.arange(NS, device=dev), top)
    first = torch.cumsum(top, 0) - top
    e = torch.arange(s_e.numel(), device=dev) - first[s_e]
    t_e = s_e // 8
    ids = f["sub_hits"][8 * start[t_e] + (s_e % 8) * n_t[t_e] + e]
    # list position of (tile, id): the point list's keys tile * P + id, sorted
    P = f["P"]
    R = int(end.max()) if T else 0
    t_j = torch.repeat_interleave(torch.arange(T, device=dev), n_t)
    keys = t_j * P + f["point_list"][:R]
    ks, kj = torch.sort(keys)
    q = t_e * P + ids
    i = torch.searchsorted(ks, q).clamp(max=max(R - 1, 0))
    assert bool((ks[i] == q).all()), "a hit-list entry is not a Gaussian of its tile's list"
    pos = kj[i] - start[t_e]
    same = s_e[1:] == s_e[:-1]
    assert bool((pos[1:][same] > pos[:-1][same]).all()), "a hit list is not in strictly increasing list position"
    # every resolved contributing pair sits at an entry below its pixel's last_entry
    Lmax = int(n_t.max()) + 1
    ekey = s_e * Lmax + pos                                   # increasing: sorted already
    pk = sid[m["pix"]] * Lmax + m["pos"]
    j = torch.searchsorted(ekey, pk).clamp(max=max(ekey.numel() - 1, 0))
    assert bool((ekey[j] == pk).all()), "a contributing pair is missing from its sub-tile's hit list"
    ent = e[j]
    assert bool((ent < le[m["pix"]]).all()), "a contributing pair lies at or beyond its pixel's last_entry"
    # the last entry of each pixel is its last contributor
    has = le > 0
    assert bool((f["n_contrib"][~has] == 0).all())
    lj = first[sid[has]] + le[has] - 1
    assert bool((pos[lj] == f["n_contrib"][has] - 1).all()), "last_entry does not end at the last contributor"

    # ---- kernel paths, block by block (render_bwd_t16_kernel) ----
    mask = torch.zeros(s_e.numel(), dtype=torch.int64, device=dev)
    mask.index_add_(0, first[sid[m["pix"]]] + ent, torch.ones_like(ent) << lane[m["pix"]])
    nblk = (top + 15) // 16
    bbase = torch.cumsum(nblk, 0) - nblk
    b = (top[s_e] - 1 - e) // 16
    blk = bbase[s_e] + b
    NB = int(nblk.sum())
    s_b = torch.repeat_interleave(torch.arange(NS, device=dev), nblk)
    b_b = torch.arange(NB, device=dev) - bbase[s_b]
    cnt = torch.clamp(top[s_b] - 16 * b_b, max=16)
    top_after = top[s_b] - 16 * b_b - cnt
    lanes_k = torch.tensor([(3 << (2 * k)) | (3 << (16 + 2 * k)) for k in range(8)], device=dev)
    le_lane = torch.zeros(NS, 32, dtype=torch.int64, device=dev)
    le_lane[sid, lane] = le
    pair_last = torch.stack([le_lane[:, [2 * k, 2 * k + 1, 16 + 2 * k, 17 + 2 * k]].amax(1) for k in range(8)], 1)
    p1_full = (pair_last[s_b].amin(1) > top_after)
    act = torch.zeros(NB, dtype=torch.int64, device=dev).index_add_(0, blk, (mask != 0).long())
    live = torch.zeros(NB, 8, dtype=torch.int64, device=dev).index_add_(0, blk, ((mask[:, None] & lanes_k) != 0).long())
    live_full = (live > 0).all(1)
    walked = act > 0
    in_image = torch.zeros(NS, dtype=torch.bool, device=dev)
    in_image[sid] = True
    return dict(phase1_full=int(p1_full.sum()), phase1_skip=int((~p1_full).sum()),
                phase2_dense=int((walked & (act + 2 >= cnt)).sum()), phase2_sparse=int((walked & (act + 2 < cnt)).sum()),
                phase3_full=int((walked & live_full).sum()), phase3_partial=int((walked & ~live_full).sum()),
                tail=int((cnt < 16).sum()), top0=int((in_image & (top == 0)).sum()))


def _saturated(f, xy, conic, op, dev, look=512):
    """Pixels where a pair after the last contributor passes the decision tests (the walk stopped at T < 1e-4), in
    float64, looking `look` positions ahead (a lower bound), and pixels that can never saturate (final_T >= 0.0102:
    T (1 - alpha) >= 1e-4 for any alpha <= 0.99)."""
    n = f["n_contrib"]
    fT = f["final_T"].double()
    never = fT >= 0.0102
    cand = torch.nonzero(~never).flatten()
    sat = torch.zeros_like(never)
    tiles_x = (W + 15) // 16
    for c in cand.split(4096):
        px, py = c % W, c // W
        tile = (py // 16) * tiles_x + px // 16
        pos = n[c][:, None] + torch.arange(look, device=dev)[None, :]
        ok = pos < (f["ranges"][tile, 1] - f["ranges"][tile, 0])[:, None]
        j = torch.where(ok, f["ranges"][tile, 0][:, None] + pos, torch.zeros_like(pos))
        gid = f["point_list"][j]
        dx = xy[gid, 0].double() - px[:, None].double()
        dy = xy[gid, 1].double() - py[:, None].double()
        pw = -0.5 * (conic[gid, 0].double() * dx * dx + conic[gid, 2].double() * dy * dy) - \
            conic[gid, 1].double() * dx * dy
        og = op[gid].double() * torch.exp(pw)
        sat[c] = (ok & (pw <= 0) & (og >= blend_f64.THR)).any(1)
    return sat, never


def _check_case(f, dev, label):
    P, ch = f["P"], f["ex"]["ch"]
    xy, conic, op, colors = blend_f64.record_fields(f["rec"])
    ex = f["ex"]
    m = blend_f64.blend(xy, conic, op, colors, f["ranges"], f["point_list"], f["n_contrib"], f["final_T"], W, H,
                        f["dpix"], torch.tensor(BG, device=dev), feat=ex.get("feat"), ex_bg=ex.get("bg"),
                        dL_dex=ex.get("dout"), image=f["color"], extra=ex.get("out"), budget=1 << 22)
    rendered = f["radii"] > 0
    used = torch.zeros(P, dtype=torch.bool, device=dev)
    used[m["gid"]] = True
    assert bool((used <= rendered).all())
    worst = torch.zeros(12, dtype=torch.float64, device=dev)
    for k, acc in enumerate(f["accs"]):
        assert bool((acc[~used] == 0).all()), f"backward {k}: a row without contributing pairs is not exactly 0"
        assert bool((acc[:, 9 + ch:] == 0).all()), f"backward {k}: slots beyond the extra channels are not 0"
        n = 9 + ch
        r = blend_f64.excess(acc[:, :n], m["a64"][:, :n], m["m64"][:, :n])
        bad = blend_f64.outside(acc[:, :n], m["a64"][:, :n], m["m64"][:, :n], TAU)
        worst[:n] = torch.maximum(worst[:n], r.amax(0))
        assert not bool(bad.any()), (f"backward {k}", int(bad.sum()), r.amax(0).tolist(),
                                     torch.nonzero(bad)[:4].tolist())
        if ch:
            d = f["dfeats"][k]
            assert torch.equal(d[rendered], acc[rendered, 9:9 + ch]) and bool((d[~rendered] == 0).all())
    # forward images
    img_r = ((f["color"].double() - m["image64"]).abs() / m["image_m"].clamp_min(1e-300)).max()
    assert bool(((f["color"].double() - m["image64"]).abs() <= TAU_IMG * m["image_m"] + 1e-30).all()), float(img_r)
    if ch:
        assert bool(((ex["out"].double() - m["extra64"]).abs() <= TAU_IMG * m["extra_m"] + 1e-30).all())
    paths = _hit_lists_and_paths(f, m, dev)
    # regimes, from the data
    sid, _ = _subtiles(dev)
    sat, never = _saturated(f, xy, conic, op, dev)
    NS = 8 * f["ranges"].shape[0]
    s_sat = torch.zeros(NS, dtype=torch.bool, device=dev).index_fill_(0, sid[sat], True)
    s_never = torch.zeros(NS, dtype=torch.bool, device=dev).index_fill_(0, sid[never], True)
    n_sub = int(torch.unique(sid).numel())
    d = f["dpix"].abs()
    dnz = d[d > 0]
    shares = dict(saturated=float(sat.double().mean()), og_past_0_99=float((m["og"] > 0.99).double().mean()),
                  near_1_255=m["near_thr"] / max(m["evaluated"], 1),
                  mixed_subtiles=float((s_sat & s_never).sum()) / n_sub, empty_subtiles=paths["top0"] / n_sub,
                  zero_cotangent=float((d.sum(0) == 0).double().mean()),
                  cotangent_decades=float(torch.log10(dnz.max() / dnz.min())))
    print(f"\n{label}: P={P} R={f['R']} longest list {int((f['ranges'][:, 1] - f['ranges'][:, 0]).max())}, "
          f"{m['pix'].numel()} contributing pairs, {m['undecided']} undecided resolved ({m['ties']} ties), "
          f"log final_T err {m['logT_err']:.1e}\n  regimes {shares}\n  paths {paths}\n"
          f"  max |a32 - a64| / m64 per slot {[f'{v:.1e}' for v in worst.tolist()]}, image {float(img_r):.1e}")
    mins = dict(saturated=0.05, og_past_0_99=2e-5, near_1_255=2e-5, mixed_subtiles=0.005, empty_subtiles=0.01,
                zero_cotangent=0.05, cotangent_decades=4.0)
    assert all(shares[k] >= v for k, v in mins.items()), shares
    assert all(v > 0 for v in paths.values()), paths
    return float(worst.max())


CASES = [  # P, extra channels, deep-list splats
    (40_000, 0, 0),
    (40_000, 1, 0),
    (40_000, 2, 0),
    (40_000, 3, 0),
    (30_000, 2, 9_000),
]


@pytest.mark.parametrize("P,ch,n_deep", CASES)
def test_blend_backward_matches_the_float64_model(cuda_device, P, ch, n_deep):
    dev = cuda_device
    cam = scenes.make_camera(W, H, device=dev)
    g = blend_regime_gaussians(P, cam, 100 + ch + n_deep, n_deep=n_deep, device=dev)
    f = _run(cam, g, ch, 7 + ch, dev)
    if n_deep:
        assert int((f["ranges"][:, 1] - f["ranges"][:, 0]).max()) > 8192
    _check_case(f, dev, f"ch={ch} n_deep={n_deep}")
