"""Float64 model of the blend, forward and backward (frosting_b200/csrc/render_fwd.cu, render_bwd.cu), pair by pair.

TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

Inputs are what the blend kernels read: the per-Gaussian record (mean2D, conic, opacity, colour as stored float32, e.g.
fb200_layout.geom_rec), the tile ranges and sorted point list, the forward's n_contrib and final_T, dL/dpixel, the
background, and optionally 1-3 extra feature channels with their background and cotangent.

Decisions.  Pixel p walks its tile's list in order; its contributing pairs are the list positions <= n_contrib[p] with
power <= 0 and alpha >= 1/255 (the T < 1e-4 stop only ever ends the walk after the last contributor).  Both tests are
evaluated in float64.  A pair is UNDECIDED when float32 could decide it the other way: |power| within K_BAND times the
float32 rounding bound of the power's three products and two sums, or op exp(power) within that bound plus the expf /
product rounding (relative) of 1/255.  Undecided pairs are resolved from the forward's own output: flipping one changes
the pixel's transmittance by a factor (1 - alpha) <= 1 - 1/255 (1 - op when the power test flips), at least 3.9e-3 in
log, while the float32 final_T is within ~1e-4 (log) of the float64 product over the same decisions (the weights below).
So every subset of a pixel's undecided pairs is tried and the one whose float64 log prod(1 - alpha) lies within
MATCH_LOG of log final_T is kept.  Subsets of equal size can only be told apart by what they blend: if several match,
the one closest to the forward's colour (and extra) image is kept, and `ties` counts such pixels.  A pixel with no
matching subset (e.g. a pair the forward culled that it should have blended) raises.  The pair at n_contrib is the
last contributor by definition and is always in.

Forward: C_p = sum_i c_i alpha_i T_i + T_f bg, T_i = prod_{j<i} (1 - alpha_j) taken as the direct product (cumprod);
the same for the extra channels with their own background.

Backward: autograd through that forward with the decision set fixed.  The reference's departures from the exact
derivative are written at the autograd level:
  * alpha = min(0.99, op G) is straight-through: alpha = og + (min(0.99, og) - og).detach();
  * slots 0/1 are d/d(NDC mean): X = X0 + 0.5 W (u - u.detach()) with u the slot's leaf (pixel = ((ndc + 1) W - 1) / 2);
  * slot 3 is half of d/d(conic.y): B = B0 + 0.5 (u - u.detach());
  * slots 9-11 are dL/d(extra feature c).
The accumulator record a64 [P,12] is returned with slots 9-11 zero beyond the channel count.

Magnitude m64 [P,12].  For pair i at pixel p, dL/dalpha_i = T_i (c_i . dp) - (sum_{j>i} alpha_j T_j (c_j . dp)
+ T_f (bg . dp)) / (1 - alpha_i) is replaced by its three parts' magnitudes
  M_i = T_i sum_c |c_ic dp_c| + (sum_{j>i} alpha_j T_j sum_c |c_jc dp_c| + T_f sum_c |bg_c dp_c|) / (1 - alpha_i)
(extra channels add their terms to each sum), and each slot's pair term by its componentwise magnitude, e.g. slot 0:
0.5 W M_i op G (|A dx| + |B dy|), slot 5: M_i G, slot 6: alpha_i T_i |dp_0|.  The float32 kernel's error on a pair term
is then a few ulp of that magnitude times the relative error of the quantities it is built from:
  * T_i and the terms behind: T is recovered from final_T by division through the pixel's n_p contributing pairs (n_p
    roundings of T, n_p of E), and final_T itself is the forward's product of the float32 (1 - alpha_j), each off by
    alpha_j / (1 - alpha_j) times alpha_j's relative error, which is (|power_j| + 4) ulp (the power's absolute error is
    about |power| ulp for an uncancelled quadratic form, expf and the opacity product add ~3 ulp).  Hence the pixel
    weight  w_p = n_p + sum_j (|power_j| + 4) alpha_j / (1 - alpha_j),  up to ~200 where two pairs clamp at 0.99;
  * the pair's own G: (|power_i| + 4) ulp, added per pair;
  * the sums: a warp adds up to 16 values per lane pair, one xor-16 add, and then one atomic add per sub-tile the
    Gaussian contributes to, in arrival order: (n_sub_g + 10) ulp of the sum of the magnitudes.
So  m64_g = sum_{pairs of g} (w_p + |power_i| + 4) |term| + (n_sub_g + 10) sum_{pairs of g} |term|,  and a float32 kernel
computing the same pairs satisfies |a32 - a64| <= tau m64 with tau a small multiple of 2^-24.  The image bound is built
the same way: m_img = sum_i (w_p + |power_i| + 4) alpha_i T_i |c_i| + w_p T_f |bg|.

Runs on whatever device the inputs are on, in chunks of pixels sorted by n_contrib so that a chunk's padded
[pixels, positions] matrices hold at most `budget` pairs (tile lists of any length fit)."""
import itertools

import torch

THR = float(torch.tensor(1.0 / 255.0, dtype=torch.float32))    # the float32 constant the kernels compare with
ULP = 2.0 ** -24
K_BAND = 16.0          # undecided band: this many times the float32 rounding bound of power / op exp(power)
MATCH_LOG = 1.5e-3     # |log prod(1 - alpha) - log final_T| of the kept decision subset (one flip is >= 3.9e-3)
MAX_UNDECIDED = 10     # per pixel


def record_fields(rec):
    """geom_rec [P,12] float32 ({x,y,conic.x,conic.y},{conic.z,opacity,r,g},{b,...}) -> (xy, conic, opacity, colors)."""
    rec = rec.reshape(-1, 12)
    return rec[:, 0:2], rec[:, 2:5], rec[:, 5], rec[:, 6:9]


def _chunks(n_sorted, budget):
    """[(lo, hi)] ranges of pixels (sorted by ascending n) with (hi - lo) * n[hi - 1] <= budget."""
    n = n_sorted.tolist()
    out, lo, N = [], 0, len(n)
    while lo < N:
        hi = lo + 1
        step = 1
        while hi < N and (hi + step - lo) * n[min(hi + step, N) - 1] <= budget:
            hi = min(hi + step, N)
            step *= 2
        while hi < N and (hi + 1 - lo) * n[hi] <= budget:
            hi += 1
        out.append((lo, hi))
        lo = hi
    return out


def blend(xy, conic, opacity, colors, ranges, point_list, n_contrib, final_T, W, H, dL_dpix, bg,
          feat=None, ex_bg=None, dL_dex=None, image=None, extra=None, budget=1 << 20):
    """The float64 blend of one frame.  Shapes: xy [P,2], conic [P,3] (x, y, z), opacity [P], colors [P,3], ranges
    [T,2], point_list [R], n_contrib / final_T [H*W] (or [H,W]), dL_dpix [3,H,W], bg [3]; feat [P,ch], ex_bg [ch],
    dL_dex [ch,H,W]; image [3,H,W] / extra [ch,H,W]: the forward's outputs, used only to break ties between equal-size
    decision subsets.  Returns a dict:
      a64, m64 [P,12]          the accumulator record and its magnitude (module docstring);
      image64, image_m [3,H,W] the colour image and its magnitude; extra64, extra_m [ch,H,W] likewise (ch = 0: empty);
      pix, pos, gid            the contributing pairs: pixel, 0-based list position, Gaussian (pixel-major, in order);
      og, power                float64 op exp(power) and power of those pairs;
      evaluated, near_thr      pairs evaluated (positions < n_contrib) and those within 1e-3 relative of 1/255;
      undecided, ties          undecided pairs resolved from final_T, pixels whose tie was broken by the image;
      logT_err                 the largest |log prod(1 - alpha) - log final_T| over all pixels."""
    dev = xy.device
    f64 = lambda t: t.detach().to(dev, torch.float64)
    P = xy.shape[0]
    ch = 0 if feat is None else feat.shape[1]
    tiles_x = (W + 15) // 16
    n_all = n_contrib.reshape(-1).to(dev, torch.int64)
    fT_all = f64(final_T.reshape(-1))
    dp = f64(dL_dpix).reshape(3, -1)
    bg = f64(bg).reshape(3)
    de = f64(dL_dex).reshape(ch, -1) if ch else None
    xb = f64(ex_bg).reshape(ch) if ch else None
    start = ranges.reshape(-1, 2)[:, 0].to(dev, torch.int64)
    plist = point_list.to(dev, torch.int64)

    # leaves: one per accumulator slot
    u = {k: f64(v).clone().requires_grad_(True) for k, v in dict(
        X=xy[:, 0], Y=xy[:, 1], A=conic[:, 0], B=conic[:, 1], C=conic[:, 2], op=opacity.reshape(-1),
        col=colors).items()}
    if ch:
        u["feat"] = f64(feat).clone().requires_grad_(True)

    HW = H * W
    image64 = torch.zeros(3, HW, dtype=torch.float64, device=dev)
    image_m = torch.zeros(3, HW, dtype=torch.float64, device=dev)
    extra64 = torch.zeros(ch, HW, dtype=torch.float64, device=dev)
    extra_m = torch.zeros(ch, HW, dtype=torch.float64, device=dev)
    m_pair = torch.zeros(P, 12, dtype=torch.float64, device=dev)     # sum of weighted pair magnitudes
    m_sum = torch.zeros(P, 12, dtype=torch.float64, device=dev)      # sum of pair magnitudes (summation term)
    img_ref = None if image is None else f64(image).reshape(3, -1)
    ex_ref = None if extra is None else f64(extra).reshape(ch, -1)
    out_pairs = {k: [] for k in ("pix", "pos", "gid", "og", "power")}
    sub_keys = []
    stats = dict(evaluated=0, near_thr=0, undecided=0, ties=0, logT_err=0.0)

    # pixels without contributors: T_f = 1, the background only
    empty = n_all == 0
    image64[:, empty] = bg[:, None] * fT_all[empty]
    image_m[:, empty] = bg.abs()[:, None] * fT_all[empty]
    if ch:
        extra64[:, empty] = xb[:, None] * fT_all[empty]
        extra_m[:, empty] = xb.abs()[:, None] * fT_all[empty]
    if bool(empty.any()):
        stats["logT_err"] = float((fT_all[empty] - 1).abs().max())

    order = torch.argsort(n_all)
    order = order[n_all[order] > 0]
    n_sorted = n_all[order]
    for lo, hi in _chunks(n_sorted.cpu(), budget):
        pc = order[lo:hi]
        nl = n_all[pc]
        R, L = pc.shape[0], int(nl.max())
        pos = torch.arange(L, device=dev)[None, :].expand(R, L)
        valid = pos < nl[:, None]
        px, py = (pc % W), (pc // W)
        tile = (py // 16) * tiles_x + px // 16
        j = torch.where(valid, start[tile][:, None] + pos, torch.zeros_like(pos))
        gid = torch.where(valid, plist[j], torch.zeros_like(pos))
        pxf, pyf = px.to(torch.float64)[:, None], py.to(torch.float64)[:, None]
        with torch.enable_grad():
            X = u["X"].detach() + 0.5 * W * (u["X"] - u["X"].detach())
            Y = u["Y"].detach() + 0.5 * H * (u["Y"] - u["Y"].detach())
            Bc = u["B"].detach() + 0.5 * (u["B"] - u["B"].detach())
            dx = X[gid] - pxf
            dy = Y[gid] - pyf
            A, B, C, op = u["A"][gid], Bc[gid], u["C"][gid], u["op"][gid]
            power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
            G = torch.exp(power)
            og = op * G
        with torch.no_grad():
            pw, ogd, opd = power.detach(), og.detach(), op.detach()
            dxd, dyd = dx.detach(), dy.detach()
            Ad, Bd, Cd = A.detach(), B.detach(), C.detach()
            e_pow = 4 * ULP * (0.5 * (Ad.abs() * dxd * dxd + Cd.abs() * dyd * dyd) + Bd.abs() * (dxd * dyd).abs()
                               + dxd.abs() * (Ad.abs() * dxd.abs() + Bd.abs() * dyd.abs())
                               + dyd.abs() * (Cd.abs() * dyd.abs() + Bd.abs() * dxd.abs()))
            band = K_BAND * (e_pow + 4 * ULP)
            pow_in, pow_out = pw < -K_BAND * e_pow, pw > K_BAND * e_pow
            og_in, og_out = ogd > THR * (1 + band), ogd < THR * (1 - band)
            dec_in = valid & pow_in & og_in
            undec = valid & ~(pow_out | og_out) & ~dec_in
            last = pos == (nl[:, None] - 1)
            bad_last = last & valid & (pow_out | og_out)
            assert not bool(bad_last.any()), "the float64 model excludes a pixel's last contributor"
            undec &= ~last
            contrib = dec_in | last
            stats["evaluated"] += int(valid.sum())
            stats["near_thr"] += int((valid & ((ogd / THR - 1).abs() <= 1e-3) & (pw <= 0)).sum())
            am = torch.minimum(ogd, torch.full_like(ogd, 0.99))
            l1 = torch.log1p(-am)
            logT = torch.where(contrib, l1, torch.zeros_like(l1)).sum(1)
            target = torch.log(fT_all[pc])
            n_und = undec.sum(1)
            rows = torch.nonzero(n_und > 0).flatten().tolist()
            stats["undecided"] += int(n_und.sum())
            for r in rows:
                ks = torch.nonzero(undec[r]).flatten().tolist()
                assert len(ks) <= MAX_UNDECIDED, (int(pc[r]), len(ks))
                lk = l1[r, ks].tolist()
                base = float(logT[r])
                tgt = float(target[r])
                match = [s for m in range(len(ks) + 1) for s in itertools.combinations(range(len(ks)), m)
                         if abs(base + sum(lk[i] for i in s) - tgt) <= MATCH_LOG]
                assert match, f"pixel {int(pc[r])}: no decision subset of its {len(ks)} undecided pairs matches final_T"
                assert len({len(s) for s in match}) == 1, f"pixel {int(pc[r])}: subsets of different sizes match"
                if len(match) > 1:
                    stats["ties"] += 1
                    match = [min(match, key=lambda s: _image_residual(r, [ks[i] for i in s], contrib, am, gid, pc,
                                                                      u, bg, xb, fT_all, img_ref, ex_ref, ch))]
                for i in match[0]:
                    contrib[r, ks[i]] = True
            logT = torch.where(contrib, l1, torch.zeros_like(l1)).sum(1)
            stats["logT_err"] = max(stats["logT_err"], float((logT - target).abs().max()))
            assert float((logT - target).abs().max()) <= MATCH_LOG, \
                f"pixel {int(pc[int((logT - target).abs().argmax())])}: the forward's final_T does not match its pairs"

        with torch.enable_grad():
            alpha = og + (torch.clamp(og, max=0.99) - og).detach()
            alpha = torch.where(contrib, alpha, torch.zeros_like(alpha))
            f = 1 - alpha
            Tin = torch.cumprod(f, 1)
            Tf = Tin[:, -1]
            T = torch.cat([torch.ones_like(Tin[:, :1]), Tin[:, :-1]], 1)
            w = alpha * T
            col = u["col"][gid]                                      # [R,L,3]
            img = torch.einsum("rl,rlc->cr", w, col) + bg[:, None] * Tf[None, :]
            loss = (img * dp[:, pc]).sum()
            if ch:
                fe = u["feat"][gid]
                ex = torch.einsum("rl,rlc->cr", w, fe) + xb[:, None] * Tf[None, :]
                loss = loss + (ex * de[:, pc]).sum()
            loss.backward()

        with torch.no_grad():
            a_, T_, w_, Tf_ = alpha.detach(), T.detach(), w.detach(), Tf.detach()
            cm = contrib.to(torch.float64)
            image64[:, pc] = img.detach()
            dpr = dp[:, pc].t()                                     # [R,3]
            cold = col.detach()
            cdp = (cold.abs() * dpr.abs()[:, None, :]).sum(2)       # [R,L]
            bgd = (bg.abs()[None, :] * dpr.abs()).sum(1)            # [R]
            if ch:
                der = de[:, pc].t()
                fed = fe.detach()
                cdp = cdp + (fed.abs() * der.abs()[:, None, :]).sum(2)
                bgd = bgd + (xb.abs()[None, :] * der.abs()).sum(1)
                extra64[:, pc] = ex.detach()
            om = 1 - a_
            wpix = nl.to(torch.float64) + ((pw.abs() + 4) * a_ / om * cm).sum(1)           # [R]
            wpair = (wpix[:, None] + pw.abs() + 4) * cm                                     # [R,L]
            wc = w_ * cdp
            behind = wc.flip(1).cumsum(1).flip(1) - wc
            Ma = (T_ * cdp + (behind + (Tf_ * bgd)[:, None]) / om) * cm
            Gd = torch.exp(pw)
            s = torch.stack([0.5 * W * Ma * ogd * (Ad.abs() * dxd.abs() + Bd.abs() * dyd.abs()),
                             0.5 * H * Ma * ogd * (Cd.abs() * dyd.abs() + Bd.abs() * dxd.abs()),
                             0.5 * Ma * ogd * dxd * dxd, 0.5 * Ma * ogd * (dxd * dyd).abs(), 0.5 * Ma * ogd * dyd * dyd,
                             Ma * Gd] + [w_ * dpr[:, c].abs()[:, None] * cm for c in range(3)] +
                            [w_ * der[:, c].abs()[:, None] * cm for c in range(ch)], -1)          # [R,L,9+ch]
            gflat = gid.reshape(-1)
            m_pair[:, :9 + ch].index_add_(0, gflat, (s * wpair[..., None]).reshape(-1, 9 + ch))
            m_sum[:, :9 + ch].index_add_(0, gflat, s.reshape(-1, 9 + ch))
            image_m[:, pc] = torch.einsum("rl,rlc->cr", w_ * wpair, cold.abs()) + \
                bg.abs()[:, None] * (Tf_ * wpix)[None, :]
            if ch:
                extra_m[:, pc] = torch.einsum("rl,rlc->cr", w_ * wpair, fed.abs()) + \
                    xb.abs()[:, None] * (Tf_ * wpix)[None, :]
            rr, ll = torch.nonzero(contrib, as_tuple=True)
            sub = ((py // 4) * ((W + 7) // 8) + px // 8)[rr]
            sub_keys.append(torch.unique(gid[rr, ll] * (((H + 3) // 4) * ((W + 7) // 8)) + sub))
            for k, v in (("pix", pc[rr]), ("pos", ll), ("gid", gid[rr, ll]), ("og", ogd[rr, ll]),
                         ("power", pw[rr, ll])):
                out_pairs[k].append(v)

    a64 = torch.zeros(P, 12, dtype=torch.float64, device=dev)
    for k, sl in (("X", 0), ("Y", 1), ("A", 2), ("B", 3), ("C", 4), ("op", 5)):
        if u[k].grad is not None:
            a64[:, sl] = u[k].grad
    if u["col"].grad is not None:
        a64[:, 6:9] = u["col"].grad
    if ch and u["feat"].grad is not None:
        a64[:, 9:9 + ch] = u["feat"].grad
    nsub = torch.zeros(P, dtype=torch.float64, device=dev)
    if sub_keys:
        keys = torch.unique(torch.cat(sub_keys))
        n_sub_tiles = ((H + 3) // 4) * ((W + 7) // 8)
        nsub.index_add_(0, keys // n_sub_tiles, torch.ones_like(keys, dtype=torch.float64))
    m64 = m_pair + (nsub + 10)[:, None] * m_sum
    # order the pair table pixel-major, positions ascending
    pairs = {k: (torch.cat(v) if v else torch.zeros(0, device=dev)) for k, v in out_pairs.items()}
    if pairs["pix"].numel():
        o = torch.argsort(pairs["pix"] * (int(pairs["pos"].max()) + 1) + pairs["pos"])
        pairs = {k: v[o] for k, v in pairs.items()}
    return dict(a64=a64, m64=m64, image64=image64.view(3, H, W), image_m=image_m.view(3, H, W),
                extra64=extra64.view(ch, H, W), extra_m=extra_m.view(ch, H, W), **pairs, **stats)


def _image_residual(r, extra_pos, contrib, am, gid, pc, u, bg, xb, fT_all, img_ref, ex_ref, ch):
    """Distance of pixel row r's float64 colour (and extra) image, with `extra_pos` added to its decided pairs, from the
    forward's image (tie-break between equal-size decision subsets)."""
    assert img_ref is not None, "equal-size decision subsets match final_T: pass the forward's image to break the tie"
    c = contrib[r].clone()
    c[extra_pos] = True
    a = torch.where(c, am[r], torch.zeros_like(am[r]))
    Tin = torch.cumprod(1 - a, 0)
    T = torch.cat([torch.ones_like(Tin[:1]), Tin[:-1]])
    w = a * T
    g = gid[r]
    p = int(pc[r])
    res = ((w[:, None] * u["col"].detach()[g]).sum(0) + bg * Tin[-1] - img_ref[:, p]).abs().sum()
    if ch:
        res = res + ((w[:, None] * u["feat"].detach()[g]).sum(0) + xb * Tin[-1] - ex_ref[:, p]).abs().sum()
    return float(res)


def excess(a32, a64, m64):
    """|a32 - a64| / m64 per element (0 where both sides are exactly 0)."""
    d = (a32.double() - a64).abs()
    return torch.where(d == 0, torch.zeros_like(d), d / m64.clamp_min(1e-300))


def outside(a32, a64, m64, tau):
    """Elements outside the bound |a32 - a64| <= tau m64 + 1e-30."""
    return (a32.double() - a64).abs() > tau * m64 + 1e-30

