"""Camera-batch driver: the per-rank render loop of a data-parallel (by camera) job (SURVEY.md 8e, 7.1 step 10).

The reference renders ONE camera per iteration on ONE GPU (frosting_trainers/refine.py:464-522: pick a camera, take
its precomputed visible-face list :487-492, render :493, loss :502-511, backward :518).  The render path shards by
camera with no data dependency between frames, so the multi-GPU form is: Gaussians replicated on every rank, the
camera batch split in contiguous blocks (one process per GPU), each rank loops over its block, and the only exchange
is the all-reduce of the scalar loss (BASELINE.json north_star).  This module is that loop as package API:

  camera_block / reduce_loss      the partition and the collective
  build_workload                  BASELINE's synthetic configs C2 / C3 / C5 (bench.py and the parity tests share them)
  visible_faces                   the per-camera visible-face sets, once, as refine.py:430-441 does
  CameraBatch                     a rank's frames: rasterizer-only, from Frosting's parameters, or a training frame
  LossReducer                     loss all-reduce off the compute stream (async NCCL work, collected every K frames)

bench.py times `CameraBatch.frame`; tests/test_bench_configs_gpu.py checks the same frames against the compiled
reference.
"""
import math
import time

import torch
import torch.distributed as dist

WORKLOADS = {
    # name: (P, W, H, sh_degree, kind, seed)   -- BASELINE.json configs
    "c3": (2_000_000, 1920, 1080, 3, "frosting", 1237),
    "c2": (500_000, 800, 800, 3, "random", 1236),
    "c5": (6_000_000, 1600, 1200, 3, "random", 1239),
    "tiny": (20_000, 320, 240, 3, "frosting", 1),
}
WORKLOAD_TEXT = {
    "c3": "C3: 2M frosting-layer Gaussians (mesh-bound prism cells, occlusion culling ON), 1920x1080, SH degree 3",
    "c2": "C2: 500k random Gaussians 800x800 SH3",
    "c5": "C5: 6M random Gaussians 1600x1200 SH3",
    "tiny": "tiny smoke workload",
}
CAMS_PER_GPU = 8
RING_RADIUS = 6.0          # SURVEY.md 8d: 64 cameras on a ring of radius 6 around the scene centre
# torch's CPU elementwise kernels round the vectorised body of each thread's chunk and its scalar tail differently
# (torch.sigmoid: a few of C3's 2 M opacities move by an ulp), so the scene's bits depend on how the tensors are split
# among intra-op threads, i.e. on torch.get_num_threads().  Scenes are generated with this fixed split, so every machine
# builds the same inputs; the reference outputs stored under tests/golden/ref were recorded with it.
SCENE_THREADS = 16


def camera_block(rank: int, world: int, n_cameras: int):
    """Contiguous block of camera indices owned by `rank` (blocks differ by at most one camera)."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    base, extra = divmod(n_cameras, world)
    start = rank * base + min(rank, extra)
    return list(range(start, start + base + (1 if rank < extra else 0)))


def reduce_loss(local_loss: torch.Tensor, group=None) -> torch.Tensor:
    """Sum of the per-rank scalar losses on every rank (NCCL over NVLink on GPUs, gloo on CPU)."""
    out = local_loss.detach().clone()
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)
    return out


class LossReducer:
    """The path's only collective, kept off the critical path.

    Every frame's scalar loss is summed over the ranks, `every` frames per collective: a frame's loss is copied into a
    device buffer (stream-ordered, no host involvement) and each full buffer goes out as ONE asynchronous all-reduce.
    The collective is ordered after the buffered losses on the device (the process group's stream waits for the current
    stream at enqueue) but the COMPUTE stream never waits for it, so a slow rank delays nobody's next frame; results are
    collected when `collect()` is called, the only point that joins the two streams.

    Why batched: a 4-byte all-reduce per frame is cheap on the wire but not on the SMs -- its kernel spins until the
    slowest rank's arrives, and with nothing idle on the GPU any more (no host wait between a frame's forward and
    backward) that spinning comes out of the blend kernels.  One collective per
    `every` frames divides it by `every`."""

    def __init__(self, group=None, every=8):
        self.group = group
        self.on = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        self.every = max(int(every), 1)
        self.buf, self.fill = None, 0
        self.pending = []

    def _flush(self):
        if self.fill == 0:
            return
        part = self.buf[:self.fill]
        work = dist.all_reduce(part, op=dist.ReduceOp.SUM, group=self.group, async_op=True) if self.on else None
        self.pending.append((part, work))
        self.buf, self.fill = None, 0

    def add(self, loss: torch.Tensor):
        if self.buf is None:
            self.buf = torch.empty(self.every, dtype=torch.float32, device=loss.device)
        self.buf[self.fill].copy_(loss.detach().reshape(()))
        self.fill += 1
        if self.fill == self.every:
            self._flush()

    def collect(self):
        """Reduced losses of every frame added since the last collect, in order, as one tensor (device)."""
        self._flush()
        out = []
        for buf, work in self.pending:
            if work is not None:
                work.wait()
            out.append(buf)
        self.pending = []
        return torch.cat(out) if out else torch.zeros(0)


def build_workload(name, device, rank=0, world=1, cams_per_gpu=CAMS_PER_GPU, ring_radius=RING_RADIUS):
    """Synthetic scene + this rank's block of the camera ring + pinned host copies of the per-frame inputs."""
    from . import scenes
    P, W, H, D, kind, seed = WORKLOADS[name]
    n_cams = cams_per_gpu * world
    cam0 = scenes.make_camera(W, H, device=device)
    block = camera_block(rank, world, n_cams)
    if kind == "frosting":
        cams = [scenes.ring_cameras(n_cams, W, H, radius=ring_radius, device=device)[i] for i in block]
    else:
        cams = [cam0] * len(block)     # free Gaussians are generated inside cam0's frustum
    wl = dict(name=name, P=P, W=W, H=H, D=D, kind=kind, cams=cams, ring_radius=ring_radius if kind == "frosting" else None)
    t = time.time()
    threads = torch.get_num_threads()
    torch.set_num_threads(SCENE_THREADS)
    try:
        if kind == "frosting":
            params, mesh = scenes.frosting_layer(P, cam0, seed, n_faces_target=max(1000, P // 2), device="cpu")
            attrs = scenes.frosting_attributes(params, mesh)
        else:
            attrs = scenes.random_gaussians(P, cam0, seed, device="cpu")
    finally:
        torch.set_num_threads(threads)
    if kind == "frosting":
        wl["mesh"] = {k: v.to(device) for k, v in mesh.items()}
        wl["params"] = {k: v.to(device) for k, v in params.items()}
    else:
        wl["mesh"] = None
    wl["attrs"] = {k: v.to(device).contiguous() for k, v in attrs.items()}
    g = torch.Generator().manual_seed(4321 + rank)
    pin = torch.cuda.is_available()
    mk = (lambda t_: t_.pin_memory()) if pin else (lambda t_: t_)
    wl["cot_host"] = [mk(torch.randn(3, H, W, generator=g)) for _ in cams]
    # per-camera host record: viewmatrix 16 | projmatrix 16 | campos 3 | bg 3 -- what Frosting builds on the CPU every
    # call and uploads (frosting_model.py:1420-1444)
    wl["cam_host"] = [mk(torch.cat([c.world_view_transform.reshape(-1).cpu(), c.full_proj_transform.reshape(-1).cpu(),
                                    c.camera_center.reshape(-1).cpu(), torch.zeros(3)]).float()) for c in cams]
    wl["face_visible"] = None
    wl["gen_s"] = time.time() - t
    return wl


def visible_faces(wl):
    """Visible-face set per camera of this rank, once (refine.py:430-441), by the CUDA prepass (row a19)."""
    from .mesh import rasterize_mesh
    if wl["mesh"] is None:
        wl["face_visible"] = None
        return None
    vis = []
    for cam in wl["cams"]:
        _, fv, _ = rasterize_mesh(wl["mesh"]["verts"], wl["mesh"]["faces"], cam.full_proj_transform,
                                  cam.image_height, cam.image_width, mark_last_on_bg=True)
        vis.append(fv.to(torch.uint8).contiguous())
    wl["face_visible"] = vis
    return vis


class CameraBatch:
    """One rank's frames over its camera block.

    mode   "raster"    inputs are the rasterizer's own tensors (the a1-a19 path): mask -> forward -> loss -> backward
           "frosting"  the frame starts from Frosting's learnable parameters (rows a20 / f1); with mask="lookup" this is
                       the single fused op `frosting_render` (sparse-row gradient contract), else attributes + rasterizer
    mask   "lookup"    occlusion culling looked up inside preprocess from the visible-face marks (`face_visibility=`): no
                       mask tensor, no mask kernel (row f1)
           "fused"     a per-Gaussian mask tensor consumed inside preprocess (`visibility_mask=`, row a19)
           "gather"    plain drop-in: Frosting's boolean gathers in torch (frosting_model.py:1578-1586) feed the rasterizer
    loss   "cot"       (color * G).sum() with a fixed random cotangent image (SURVEY.md 8d "frame")
           "l1_dssim"  0.8 L1 + 0.2 (1 - SSIM) against a ground-truth image (refine.py:407-409), fused kernel (row f2)
    """

    def __init__(self, wl, device, mode="raster", mask="lookup", loss="cot", optimizer=None):
        import frosting_b200 as fb
        from . import scenes
        self.fb, self.scenes, self.wl, self.device = fb, scenes, wl, device
        self.mode, self.mask_mode, self.loss_mode = mode, mask, loss
        self.P = wl["P"]
        self.opt = optimizer
        if mode == "raster":
            self.leaves = {k: v.clone().requires_grad_(True) for k, v in wl["attrs"].items()}
        elif optimizer is not None:
            self.params = optimizer.params
        else:
            self.params = {k: v.clone().requires_grad_(True) for k, v in wl["params"].items()}
        self.gt = None
        if wl["mesh"] is not None and wl.get("face_visible") is None:
            visible_faces(wl)

    def settings(self, cam):
        return self.scenes.settings_for(cam, self.wl["D"], device=self.device)

    def render_mask(self, i):
        if self.wl["face_visible"] is None:
            return None
        return self.fb.gaussian_render_mask(self.wl["face_visible"][i], self.wl["mesh"]["cells"], self.P)

    def frame(self, i, rs, cot):
        """forward + loss + backward of camera i of this rank; returns the detached scalar loss."""
        fb = self.fb
        lookup = self.mask_mode == "lookup" and self.wl["face_visible"] is not None
        mask = None if lookup else self.render_mask(i)
        fv = self.wl["face_visible"][i] if lookup else None
        if self.mode == "frosting" and (lookup or self.wl["face_visible"] is None):
            if self.opt is None:
                for v in self.params.values():
                    v.grad = None
            color, radii = fb.frosting_render(self.params, self.wl["mesh"], rs, face_visible=fv,
                                              grad_sink=self.opt.grads if self.opt is not None else None)
            loss = fb.l1_dssim_loss(color, self.gt[i], 0.2) if self.loss_mode == "l1_dssim" else (color * cot).sum()
            loss.backward()
            self.last = dict(color=color, radii=radii, means2D=None)
            return loss.detach()
        if self.mode == "raster":
            L = self.leaves
            for v in L.values():
                v.grad = None                                        # zero_grad(set_to_none=True), refine.py:522
            a = L
        else:
            if self.opt is None:
                for v in self.params.values():
                    v.grad = None
            a = fb.frosting_attributes_fused(self.params, self.wl["mesh"], mask,
                                             grad_sink=self.opt.grads if self.opt is not None else None, face_visible=fv)
        if mask is not None and self.mask_mode == "gather":
            keep = mask.bool()
            m3, op, sh, sc, ro = (a[k][keep] for k in ("means3D", "opacities", "shs", "scales", "rotations"))
            means2D = torch.zeros_like(m3, requires_grad=True)       # frosting_model.py:1624
            color, radii = fb.GaussianRasterizer(rs)(means3D=m3, means2D=means2D, opacities=op, shs=sh, scales=sc,
                                                     rotations=ro)
        else:
            means2D = torch.zeros(self.P, 3, device=self.device, requires_grad=True)
            color, radii = fb.GaussianRasterizer(rs)(
                means3D=a["means3D"], means2D=means2D, opacities=a["opacities"], shs=a["shs"], scales=a["scales"],
                rotations=a["rotations"], visibility_mask=mask,
                face_visibility=(fv, self.wl["mesh"]["cells"]) if lookup else None)
        if self.loss_mode == "l1_dssim":
            loss = fb.l1_dssim_loss(color, self.gt[i], 0.2)
        else:
            loss = (color * cot).sum()
        loss.backward()
        self.last = dict(color=color, radii=radii, means2D=means2D)
        return loss.detach()

    def run(self, steps, rs_list, cot_list, reducer=None, start=0):
        """`steps` frames cycling over this rank's cameras; the losses go through `reducer` (LossReducer) if given."""
        n = len(self.wl["cams"])
        for k in range(steps):
            i = (start + k) % n
            loss = self.frame(i, rs_list[i], cot_list[i])
            if reducer is not None:
                reducer.add(loss)
        return reducer.collect() if reducer is not None else None
