"""The per-tile sort (binning.cu) against its specification, not against the reference: every tile's segment holds the
keys (depth_bits << 32 | gaussian_idx) of exactly the Gaussians whose tile rectangle covers the tile, in strictly
increasing order, and point_list holds their low 32 bits.  The inputs send tiles of the tiny and medium size classes
through both of their algorithms: the bucket sort (continuous depths) and the radix fallback (every Gaussian on one of
three depths, so with more than 3 x 24 keys some bucket overflows)."""
import numpy as np
import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import scenes

pytestmark = pytest.mark.gpu

CLASSES = (("tiny", 512), ("small", 2048), ("medium", 8192))   # longest list of each shared-memory class = its buckets
INSERT_MAX = 24                                                 # fullest bucket the bucket sort finishes by insertion


def sort_path(depth_bits):
    """(size class, algorithm) that binning.cu runs on a tile whose keys have these depth bits."""
    n = len(depth_bits)
    if n == 1:
        return "tiny", "none"
    for name, buckets in CLASSES:
        if n <= buckets:
            break
    else:
        return "global", "radix"
    d = depth_bits.astype(np.int64)
    shift = max(0, int(d.max() - d.min()).bit_length() - (buckets.bit_length() - 1))
    fullest = int(np.bincount((d - d.min()) >> shift).max())
    return name, ("radix" if fullest > INSERT_MAX else "bucket")


def check_tiles(st, W, H):
    """Asserts the specification on every tile of a forward_with_state result; returns the sort paths taken."""
    tiles_x = (W + 15) // 16
    count = st["tile_count"].long().cpu()
    ranges = st["ranges"].long().cpu()
    start = torch.cumsum(count, 0) - count
    used = count > 0
    assert torch.equal(ranges[used, 0], start[used]) and torch.equal(ranges[used, 1], (start + count)[used])
    assert int(ranges[~used].abs().sum()) == 0, "empty tiles keep the range (0, 0)"
    assert st["num_rendered"] == int(count.sum())
    keys = st["keys"].cpu()
    assert torch.equal(st["point_list"].cpu(), (keys & 0xffffffff).int())
    depth_bits = st["depth"].cpu().view(torch.int32).long()
    rect = st["rect"].cpu().long()
    minx, miny = rect[:, 0] & 0xffff, (rect[:, 0] >> 16) & 0xffff
    maxx, maxy = rect[:, 1] & 0xffff, (rect[:, 1] >> 16) & 0xffff
    paths = set()
    for t in torch.nonzero(used).flatten().tolist():
        seg = keys[start[t]:start[t] + count[t]]
        ids = seg & 0xffffffff
        assert bool((seg[1:] > seg[:-1]).all()), f"tile {t}: keys not strictly increasing"
        assert torch.equal(seg >> 32, depth_bits[ids]), f"tile {t}: key depth bits differ from the Gaussians' depths"
        tx, ty = t % tiles_x, t // tiles_x
        covers = torch.nonzero((minx <= tx) & (tx < maxx) & (miny <= ty) & (ty < maxy)).flatten()
        assert torch.equal(torch.sort(ids).values, covers), f"tile {t}: not the Gaussians whose rectangle covers it"
        paths.add(sort_path((seg >> 32).numpy()))
    return paths


CASES = [
    # class, algorithm, P, W, H, scale multiplier, depths (None: continuous)
    ("tiny", "bucket", 6_000, 128, 96, 1.0, None),
    ("tiny", "radix", 6_000, 128, 96, 1.0, (4.0, 5.0, 6.0)),
    ("medium", "bucket", 9_000, 64, 48, 3.0, None),
    ("medium", "radix", 9_000, 64, 48, 3.0, (4.0, 5.0, 6.0)),
]


def case_inputs(P, W, H, scale, depths, device):
    cam = scenes.make_camera(W, H, device=device)
    g = scenes.random_gaussians(P, cam, 31, device=device, large_frac=0.0, near_frac=0.0)
    g["scales"] = g["scales"] * scale
    if depths is not None:           # slide every Gaussian along its ray onto one of the given depths
        z = torch.tensor(depths, device=device).repeat(P // len(depths) + 1)[:P]
        g["means3D"][:, :2] *= (z / g["means3D"][:, 2])[:, None]
        g["means3D"][:, 2] = z
    return cam, g


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}_{c[1]}")
def test_tile_sort_meets_specification(case, cuda_device):
    cls, algo, P, W, H, scale, depths = case
    cam, g = case_inputs(P, W, H, scale, depths, cuda_device)
    rs = scenes.settings_for(cam, 0, device=cuda_device)
    st = fb.forward_with_state(rs, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"],
                               rotations=g["rotations"])
    paths = check_tiles(st, W, H)
    assert (cls, algo) in paths, paths
