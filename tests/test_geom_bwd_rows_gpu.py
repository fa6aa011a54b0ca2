"""SH rows of every width through the per-Gaussian backward's in-place walk (the dense gradient contract).

Rows of 1, 9 and 20 coefficients must give the frame of the same scene with 16-coefficient rows at the same degree:
the same image and radii, gradients equal up to the order of the blend backward's float atomics, exact zeros for the
coefficients at or beyond (D+1)^2.  P is not a multiple of 32 and the scene's last Gaussians sit behind the camera, so
the final, shorter run of 32 rows has nothing rendered.  Every gradient buffer starts as NaN: a row the backward does
not write shows up."""
import ctypes as C

import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import _lib
from frosting_b200._lib import Grads
from tests.test_c_abi_gpu import _one_phase, _p
from tests.util import scene, rel_err_stats

pytestmark = pytest.mark.gpu

P, W, H = 30_013, 320, 208      # P % 32 == 29
N_BEHIND = 64


def _frame(rs, g, D, dev):
    """Forward and dense backward straight through the C ABI."""
    R = fb.forward_with_state(rs, g["means3D"], g["opacities"], shs=g["shs"], scales=g["scales"],
                              rotations=g["rotations"])["num_rendered"]
    prm, inp, ws, color, radii, st, keep = _one_phase(rs, g, P, W, H, D, R + 17, dev)
    assert st[_lib.ST_OVERFLOW] == 0
    M = g["shs"].shape[1]
    nan = lambda *shape: torch.full(shape, float("nan"), device=dev)
    out = dict(means2D=nan(P, 3), opacities=nan(P, 1), means3D=nan(P, 3), shs=nan(P, M, 3), scales=nan(P, 3),
               rotations=nan(P, 4))
    grads = Grads(d_dL_dmeans2D=_p(out["means2D"]), d_dL_dcolors=None, d_dL_dopacity=_p(out["opacities"]),
                  d_dL_dmeans3D=_p(out["means3D"]), d_dL_dcov3D=None, d_dL_dsh=_p(out["shs"]),
                  d_dL_dscales=_p(out["scales"]), d_dL_drotations=_p(out["rotations"]))
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(4)).to(dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(_lib.lib().fb200_backward(C.byref(prm), C.byref(inp), C.byref(ws), _p(radii), _p(cot), C.byref(grads),
                                         stream))
    torch.cuda.synchronize(dev)
    return color, radii, out


@pytest.mark.parametrize("M,D", [(1, 0), (9, 2), (20, 3)])
def test_sh_rows_of_every_width_match_16_coefficient_rows(cuda_device, M, D):
    dev = cuda_device
    cam, g, rs = scene(P, W, H, 5, D, dev)
    # p_view = [p, 1] @ viewmatrix: the last Gaussians at view depth -5
    behind = torch.tensor([0.0, 0.0, -5.0, 1.0], dtype=torch.float64) @ torch.linalg.inv(rs.viewmatrix.cpu().double())
    g["means3D"][-N_BEHIND:] = behind[:3].float().to(dev)
    sh16 = g["shs"]
    if M <= 16:
        shM = sh16[:, :M].contiguous()
    else:
        shM = torch.cat([sh16, torch.randn(P, M - 16, 3, generator=torch.Generator().manual_seed(6)).to(dev)], 1)
    c16, r16, o16 = _frame(rs, g, D, dev)
    cM, rM, oM = _frame(rs, dict(g, shs=shM), D, dev)
    assert torch.equal(rM, r16) and torch.equal(cM.view(torch.int32), c16.view(torch.int32))
    dead = r16 <= 0
    assert P % 32 != 0 and bool(dead[-N_BEHIND:].all()) and int((~dead).sum()) > 0
    ncoef = (D + 1) * (D + 1)
    for out in (o16, oM):
        for k, v in out.items():
            assert bool(torch.isfinite(v).all()), k
            assert float(v[dead].abs().sum()) == 0.0, k
        assert float(out["shs"][:, ncoef:].abs().sum()) == 0.0
    for k in o16:
        mine, ref = oM[k], o16[k]
        if k == "shs":
            mine, ref = mine[:, :ncoef], ref[:, :ncoef]
        m, _ = rel_err_stats(mine, ref)
        assert m <= 1e-3, (k, m)      # two frames: the blend backward's float atomics sum in different orders
