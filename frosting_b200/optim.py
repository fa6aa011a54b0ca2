"""Data-parallel Adam for camera-sharded Frosting training (SURVEY.md row f3) -- host side.

Mirrors the reference's optimizer wrapper (frosting_scene/frosting_optimizer.py): `OptimizationParams` carries the
same defaults (:7-36), `FrostingAdam` exposes `step / zero_grad / update_learning_rate / state_dict` with the same
group names and learning rates (:74-101) and the same two exponential schedules (:103-114, 123-134).  What is new is
where the numbers live and how ranks exchange them:

* all learnable tensors are views into ONE flat fp32 parameter slab, their gradients views into ONE gradient slab
  (`FlatSlabs`); the fused attribute backward (`frosting_attributes_fused(..., grad_sink=opt.grads)`) writes straight
  into the gradient slab, so there is no `.grad` accumulation pass;
* under `torch.distributed` with world > 1 both slabs are peer-mapped (torch symmetric memory, else cudaIpc handles
  exchanged once through `all_gather_object`) and `step()` launches `fb200_adam_step`: each rank reduces ITS 1/world shard of the gradients
  out of all ranks' slabs over NVLink, updates its shard of the Adam moments, and stores the new parameters into
  every rank's slab -- gradient all-reduce, optimizer and parameter broadcast in one kernel; at 4 ranks the sum
  is formed in the NVSwitch (multimem.ld_reduce on the slabs' multicast mapping) and the parameters are broadcast by
  it (multimem.st).  The two rendezvous it needs are 4-byte NCCL all-reduces (the first one carries the scalar loss);
* world == 1: the same kernel as a plain fused multi-group Adam.

There is no CPU path: the slabs are CUDA memory and the step is the CUDA kernel.
"""
import ctypes as C
import math

import numpy as np
import torch
import torch.distributed as dist

from . import _lib


class OptimizationParams:
    """Same fields and defaults as frosting_scene/frosting_optimizer.py:7-36."""

    def __init__(self, iterations=30_000, position_lr_init=0.00016, position_lr_final=0.0000016,
                 position_bary_coords_lr_init=0.005, position_bary_coords_lr_final=0.00005,
                 position_lr_delay_mult=0.01, position_lr_max_steps=30_000, feature_lr=0.0025, opacity_lr=0.05,
                 scaling_lr=0.005, rotation_lr=0.001):
        self.iterations = iterations
        self.position_lr_init = position_lr_init
        self.position_lr_final = position_lr_final
        self.position_bary_coords_lr_init = position_bary_coords_lr_init
        self.position_bary_coords_lr_final = position_bary_coords_lr_final
        self.position_lr_delay_mult = position_lr_delay_mult
        self.position_lr_max_steps = position_lr_max_steps
        self.feature_lr = feature_lr
        self.opacity_lr = opacity_lr
        self.scaling_lr = scaling_lr
        self.rotation_lr = rotation_lr


def get_expon_lr_func(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """Log-linear interpolation lr_init -> lr_final over max_steps with an optional sine warm-up
    (frosting_utils/general_utils.py:23-56)."""

    def at(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        delay = 1.0
        if lr_delay_steps > 0:
            delay = lr_delay_mult + (1 - lr_delay_mult) * math.sin(0.5 * math.pi * min(max(step / lr_delay_steps, 0), 1))
        t = min(max(step / max_steps, 0), 1)
        return delay * math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)

    return at


# ---- slab layout (pure host logic; covered on CPU by tests/test_host_logic_cpu.py) ----

def slab_layout(sizes, world=1):
    """Element offsets of consecutive groups of `sizes` elements, each start rounded up to 4 elements (16 B), and the
    padded total (a multiple of 4 * world so that equal shards are 4-aligned).  Returns (starts[len+1], total)."""
    starts, at = [], 0
    for n in sizes:
        if n < 0:
            raise ValueError("negative group size")
        starts.append(at)
        at += (int(n) + 3) // 4 * 4
    quantum = 4 * max(int(world), 1)
    total = (at + quantum - 1) // quantum * quantum
    starts.append(at)
    return starts, total


def shard_range(total, rank, world):
    """[lo, hi) of the flat slab owned by `rank`: equal 4-aligned shards (total is a multiple of 4 * world)."""
    if total % (4 * world):
        raise ValueError("total must be a multiple of 4 * world")
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    per = total // world
    return rank * per, (rank + 1) * per


class _DevicePointer:
    """`__cuda_array_interface__` carrier so torch can view memory this library allocated."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (int(ptr), False), "version": 2}


def _view(ptr, n, device):
    return torch.as_tensor(_DevicePointer(ptr, n), device=device)


class GradSink(dict):
    """name -> view into the gradient slab, plus the book-keeping torch keeps in `.grad is None`: which groups have
    a gradient this step.  Fetching a view (`sink[name]`) declares that the group receives one -- every producer
    gets its destination that way -- and `step()` skips the groups nobody fetched since the last step / zero_grad.
    Producers OVERWRITE their views (one write per element, no read-modify-write), so a second fused backward into
    the sink before the step would silently drop the first: `sink_once` raises instead."""

    accepts_row_radii = False     # set per instance by FlatSlabs(rows=...)

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.written = set()
        self.sunk = set()
        # sparse-row producers (frosting_render): `row_radii` [rows] int32 of the frame that wrote the views named in
        # `sparse_names`; rows with radii <= 0 are zero rows that were NOT written and must not be read
        self.row_radii = None
        self.sparse_names = set()

    def rows_from(self, radii, names):
        if not self.accepts_row_radii:
            raise RuntimeError("this gradient sink has no row structure: zero-fill instead")
        self.row_radii = radii
        self.sparse_names |= set(names)

    def __getitem__(self, name):
        self.written.add(name)
        return super().__getitem__(name)

    def sink_once(self, names):
        names = set(names)
        twice = names & self.sunk
        if twice:
            raise RuntimeError(
                f"gradient slab views {sorted(twice)} written twice between optimizer steps: producers overwrite, they do "
                "not accumulate -- sum the losses of the cameras into one backward, or step between them")
        self.sunk |= names

    def clear(self):   # not dict.clear: the views stay
        self.written = set()
        self.sunk = set()
        self.row_radii = None
        self.sparse_names = set()


class FlatSlabs:
    """Parameter and gradient slabs + named views.  `tensors`: ordered dict name -> initial CUDA tensor."""

    def __init__(self, tensors, world=1, rank=0, peer=False, group=None, rows=None, row_names=None):
        """`rows`: when given, tensors whose first dimension equals it are row-structured (one row per Gaussian) and the
        gradient slab carries a [rows] int32 radii region behind the gradients -- peer-visible like the slab itself --
        through which a sparse-row producer tells every rank's step which of ITS rows exist (fb200_adam_args.peer_row_radii).
        `row_names`: the row-structured tensors named explicitly (default: every tensor whose first dimension is `rows`;
        a tensor that only happens to have that many rows -- Frosting's background Gaussians -- must not count)."""
        names = list(tensors)
        first = tensors[names[0]]
        if not first.is_cuda:
            raise RuntimeError("frosting_b200 optimizers keep their state in CUDA memory (no CPU fallback)")
        self.device, self.names, self.world, self.rank, self.group = first.device, names, world, rank, group
        self.shapes = {n: tuple(tensors[n].shape) for n in names}
        self.starts, self.total = slab_layout([tensors[n].numel() for n in names], world)
        self.rows = int(rows) if rows else 0
        self.row_width = [tensors[n].numel() // self.rows if self.rows and tensors[n].dim() >= 1 and
                          tensors[n].shape[0] == self.rows and (row_names is None or n in row_names) else 0
                          for n in names]
        self.alloc = self.total + (self.rows + 3) // 4 * 4       # elements allocated per slab: Adam's range + the radii region
        self._owned, self._opened = [], []
        self.mc_params = self.mc_grads = 0      # NVSwitch multicast mappings of the two slabs (0: none)
        self.transport = "local"
        L = _lib.lib()
        if peer and self._try_symmetric():
            pass
        elif peer:
            with torch.cuda.device(self.device):
                ptrs = []
                for _ in range(2):
                    p = C.c_void_p()
                    _lib.check(L.fb200_peer_alloc(self.alloc * 4, C.byref(p)))
                    self._owned.append(p.value)
                    ptrs.append(p.value)
                self.param_slab = _view(ptrs[0], self.alloc, self.device)
                self.grad_slab = _view(ptrs[1], self.alloc, self.device)
                self.peer_params, self.peer_grads = self._exchange(L, ptrs)
                self.transport = "cudaIpc peer pointers"
        else:
            self.param_slab = torch.zeros(self.alloc, dtype=torch.float32, device=self.device)
            self.grad_slab = torch.zeros(self.alloc, dtype=torch.float32, device=self.device)
            self.peer_params, self.peer_grads = [self.param_slab.data_ptr()], [self.grad_slab.data_ptr()]
        self.params, self.grads = {}, GradSink()
        self.row_radii = None
        if self.rows:
            # sparse gradient rows pay off on the local and peer-pointer paths (a peer's vector is fetched only where it
            # rendered something); the in-switch sum cannot skip rows and is taken from 4 ranks up -- there the producer
            # zero-fills instead
            self.grads.accepts_row_radii = not (self.mc_params and self.mc_grads)
            self.row_radii = self.grad_slab[self.total:self.total + self.rows].view(torch.int32)
        for n, s in zip(names, self.starts):
            k = tensors[n].numel()
            self.param_slab[s:s + k].copy_(tensors[n].detach().reshape(-1).to(torch.float32))
            self.params[n] = self.param_slab[s:s + k].view(self.shapes[n]).requires_grad_(True)
            self.grads[n] = self.grad_slab[s:s + k].view(self.shapes[n])

    def _try_symmetric(self):
        """Slabs in torch symmetric memory: peer pointers for every rank AND, on an NVSwitch box, one multicast
        mapping per slab, which lets the step reduce the gradients in the switch (multimem.ld_reduce) and broadcast
        the parameters through it (multimem.st).  Every rank must take the same branch, so the outcome is agreed on
        with an all-reduce; any failure falls back to cudaIpc peer pointers (still CUDA, still one fused kernel)."""
        import os
        ok, slabs, handles = 1, [], []
        # symmetric memory (peer pointers at 2 ranks, in-switch reduction from 4 up); FB200_NO_SYMM_MEM=1 forces the
        # cudaIpc path
        if os.environ.get("FB200_NO_SYMM_MEM"):
            ok = 0
        else:
            try:
                import torch.distributed._symmetric_memory as symm
                group = self.group if self.group is not None else dist.group.WORLD
                with torch.cuda.device(self.device):
                    for _ in range(2):
                        t = symm.empty(self.alloc, dtype=torch.float32, device=self.device)
                        t.zero_()
                        slabs.append(t)
                    torch.cuda.synchronize(self.device)
                    for t in slabs:
                        handles.append(symm.rendezvous(t, group=group.group_name))
            except Exception as ex:   # unsupported build / driver / topology
                self._symm_error = repr(ex)
                ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            return False
        self._symm_keep = (slabs, handles)
        self.param_slab, self.grad_slab = slabs
        out = []
        for t, h in zip(slabs, handles):
            base = [int(x) for x in h.buffer_ptrs]
            off = t.data_ptr() - base[self.rank]            # the tensor's offset inside the symmetric allocation
            mc = int(getattr(h, "multicast_ptr", 0) or 0)
            out.append(([b + off for b in base], mc + off if mc else 0))
        (self.peer_params, self.mc_params), (self.peer_grads, self.mc_grads) = out
        # multicast must be available on every rank for both slabs
        flag = torch.tensor([1 if (self.mc_params and self.mc_grads) else 0], dtype=torch.int32, device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        # the in-switch path costs about the same whatever the world size, the peer-pointer path grows with it; multicast
        # from 4 ranks up (the crossover has not been re-measured on H100 NVSwitch boxes)
        want_mc = self.world >= 4 if not os.environ.get("FB200_MULTICAST") else os.environ["FB200_MULTICAST"] == "1"
        if int(flag.item()) == 0 or not want_mc:
            self.mc_params = self.mc_grads = 0
            self.transport = "symmetric-memory peer pointers"
        else:
            self.transport = "NVSwitch multicast (multimem.ld_reduce / multimem.st)"
        return True

    def _exchange(self, L, ptrs):
        """Trade cudaIpc handles with the other ranks of the box and map their slabs."""
        mine = []
        for p in ptrs:
            h = C.create_string_buffer(_lib.PEER_HANDLE_BYTES)
            _lib.check(L.fb200_peer_export(C.c_void_p(p), h))
            mine.append(h.raw)
        everyone = [None] * self.world
        dist.all_gather_object(everyone, mine, group=self.group)
        out = ([], [])
        for r, handles in enumerate(everyone):
            for which, h in enumerate(handles):
                if r == self.rank:
                    out[which].append(ptrs[which])
                    continue
                q = C.c_void_p()
                _lib.check(L.fb200_peer_open(h, C.byref(q)))
                self._opened.append(q.value)
                out[which].append(q.value)
        return out

    def close(self):
        """Unmap peers and free the slabs (all ranks must have stopped using them: call after a barrier)."""
        L = _lib.lib()
        with torch.cuda.device(self.device):
            torch.cuda.synchronize(self.device)
            for q in self._opened:
                L.fb200_peer_close(C.c_void_p(q))
            for p in self._owned:
                L.fb200_peer_free(C.c_void_p(p))
        self._opened, self._owned = [], []
        self._symm_keep = None


class FrostingAdam:
    """Adam(lr per group, eps=1e-15) over flat slabs, data-parallel over the ranks of one box.

    `tensors`: ordered dict name -> initial CUDA tensor; `lrs`: dict name -> learning rate.  After construction use
    `opt.params[name]` as the learnable tensors (views into the parameter slab) and route gradients into
    `opt.grads[name]` (views into the gradient slab; `frosting_attributes_fused(..., grad_sink=opt.grads)` does that
    in its backward; `opt.collect_grads()` copies autograd's `.grad` there for any other producer -- `step()` does it
    itself when nothing was written).  `state_dict()` / `load_state_dict()` speak torch.optim.Adam's format."""

    def __init__(self, tensors, lrs, betas=(0.9, 0.999), eps=1e-15, group=None, average=True, rows=None, row_names=None):
        if len(tensors) > _lib.ADAM_MAX_GROUPS:
            raise ValueError(f"at most {_lib.ADAM_MAX_GROUPS} parameter groups")
        self.group = group
        distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if distributed else 1
        self.rank = dist.get_rank(group) if distributed else 0
        if self.world > _lib.MAX_PEERS:
            raise ValueError(f"at most {_lib.MAX_PEERS} ranks (one NVSwitch box)")
        self.slabs = FlatSlabs(tensors, self.world, self.rank, peer=self.world > 1, group=group, rows=rows,
                               row_names=row_names)
        self.params, self.grads = self.slabs.params, self.slabs.grads
        self.param_groups = [{"name": n, "lr": float(lrs[n]), "params": [self.params[n]]} for n in self.slabs.names]
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        self.grad_scale = 1.0 / self.world if average else 1.0
        self.lo, self.hi = shard_range(self.slabs.total, self.rank, self.world)
        dev = self.slabs.device
        self.exp_avg = torch.zeros(self.hi - self.lo, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(self.hi - self.lo, dtype=torch.float32, device=dev)
        self.current_iteration = 0
        self._flag = torch.zeros(1, dtype=torch.float32, device=dev)
        self.position_sheduler_func = None
        self.position_bary_coords_sheduler_func = None

    # -- the reference's group list and schedules (frosting_optimizer.py:74-114) for the Frosting layer's tensors --
    GROUP_OF = {"bary_logits": "bary_coords", "sh_dc": "sh_coordinates_dc", "sh_rest": "sh_coordinates_rest",
                "opacity_logits": "opacities", "log_scales": "scales", "quats": "quaternions",
                "bg_points": "bg_points", "bg_opacity_logits": "bg_opacities", "bg_sh_dc": "bg_sh_coordinates_dc",
                "bg_sh_rest": "bg_sh_coordinates_rest", "bg_log_scales": "bg_scales", "bg_quats": "bg_quaternions"}

    @classmethod
    def for_frosting(cls, params, opt=None, spatial_lr_scale=1.0, group=None):
        opt = opt or OptimizationParams()
        order = ("bary_logits", "sh_dc", "sh_rest", "opacity_logits", "log_scales", "quats")
        lr = {"bary_logits": opt.position_bary_coords_lr_init, "sh_dc": opt.feature_lr, "sh_rest": opt.feature_lr / 20.0,
              "opacity_logits": opt.opacity_lr, "log_scales": opt.scaling_lr, "quats": opt.rotation_lr}
        mesh_order = order
        if "bg_points" in params:
            # background Gaussians: the reference's six extra groups, in its order (frosting_optimizer.py:86-92)
            order = order + ("bg_points", "bg_opacity_logits", "bg_sh_dc", "bg_sh_rest", "bg_log_scales", "bg_quats")
            lr.update({"bg_points": opt.position_lr_init * spatial_lr_scale, "bg_opacity_logits": opt.opacity_lr,
                       "bg_sh_dc": opt.feature_lr, "bg_sh_rest": opt.feature_lr / 20.0, "bg_log_scales": opt.scaling_lr,
                       "bg_quats": opt.rotation_lr})
        # one row per mesh-bound Gaussian in each of the six mesh tensors: `frosting_render` writes the rendered rows only
        # and hands `radii` over; the background groups are dense (zero-filled rows)
        self = cls({n: params[n] for n in order}, lr, eps=1e-15, group=group, rows=params["bary_logits"].shape[0],
                   row_names=mesh_order)
        for g in self.param_groups:
            g["name"] = cls.GROUP_OF[g["name"]]
        self.num_iterations = opt.iterations
        self.spatial_lr_scale = spatial_lr_scale
        self.position_sheduler_func = get_expon_lr_func(opt.position_lr_init * spatial_lr_scale,
                                                        opt.position_lr_final * spatial_lr_scale,
                                                        lr_delay_mult=opt.position_lr_delay_mult,
                                                        max_steps=opt.position_lr_max_steps)
        self.position_bary_coords_sheduler_func = get_expon_lr_func(opt.position_bary_coords_lr_init,
                                                                    opt.position_bary_coords_lr_final,
                                                                    lr_delay_mult=opt.position_lr_delay_mult,
                                                                    max_steps=opt.position_lr_max_steps)
        return self

    def update_learning_rate(self, iteration=None):
        """frosting_optimizer.py:123-134."""
        if iteration is None:
            iteration = self.current_iteration
        lr = 0.0
        for g in self.param_groups:
            if g["name"] in ("shell_base_verts", "inner_dist", "outer_dist", "bg_points") and self.position_sheduler_func:
                lr = self.position_sheduler_func(iteration)
                g["lr"] = lr
            if g["name"] == "bary_coords" and self.position_bary_coords_sheduler_func:
                lr = self.position_bary_coords_sheduler_func(iteration)
                g["lr"] = lr
        return lr

    def zero_grad(self, set_to_none=True):
        """torch semantics with set_to_none=True (what the reference calls, refine.py:522): every group is back to "no
        gradient"; a group that receives none before the next step is SKIPPED by it (moments, parameters untouched), as
        torch.optim.Adam skips parameters whose .grad is None.  Nothing is cleared on the device: producers overwrite their
        views, and an unwritten view is never read.  set_to_none=False zero-fills the slab and marks every group written
        (torch then steps them with a zero gradient)."""
        for p in self.params.values():
            p.grad = None
        self.grads.clear()
        if not set_to_none:
            self.slabs.grad_slab.zero_()
            self.grads.written = set(self.slabs.names)

    def collect_grads(self):
        """Copy autograd-populated `.grad`s into the gradient slab (for producers that do not take `grad_sink`)."""
        for n, p in list(self.params.items()):
            if p.grad is not None:
                self.grads[n].copy_(p.grad)

    def _args(self):
        t = self.current_iteration
        a = _lib.AdamArgs()
        a.world, a.rank = self.world, self.rank
        for r in range(self.world):
            a.peer_params[r] = self.slabs.peer_params[r]
            a.peer_grads[r] = self.slabs.peer_grads[r]
        a.d_exp_avg, a.d_exp_avg_sq = self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr()
        a.shard_lo, a.shard_hi = self.lo, self.hi
        a.n_groups = len(self.param_groups)
        for k, s in enumerate(self.slabs.starts[:-1]):
            a.group_start[k] = s
            # a group without a gradient this step is skipped entirely (negative lr = the kernel's "skip" mark); with
            # world > 1 every rank must have written the same groups, which holds for replicas running the same graph
            a.lr[k] = self.param_groups[k]["lr"] if self.slabs.names[k] in self.grads.written else -1.0
        a.group_start[a.n_groups] = self.slabs.total
        b1, b2 = self.betas
        a.beta1, a.beta2, a.eps = b1, b2, self.eps
        a.bias_correction1 = 1.0 - b1 ** t
        a.bias_correction2_sqrt = math.sqrt(1.0 - b2 ** t)
        a.grad_scale = self.grad_scale
        a.mc_grads = self.slabs.mc_grads or None
        a.mc_params = self.slabs.mc_params or None
        if self.grads.row_radii is not None:
            # sparse gradient rows: every rank's radii sit behind its gradient slab, so the peer mappings cover them
            for r in range(self.world):
                a.peer_row_radii[r] = self.slabs.peer_grads[r] + 4 * self.slabs.total
            for k, n in enumerate(self.slabs.names):
                a.row_width[k] = self.slabs.row_width[k] if n in self.grads.sparse_names else 0
            a.row_count = self.slabs.rows
        return a

    def step(self, loss=None):
        """One optimizer step on the current stream.  `loss` (optional CUDA scalar): summed over ranks in place by the
        first rendezvous, as the training loop's loss all-reduce."""
        self.current_iteration += 1
        dev = self.slabs.device
        if not self.grads.written:
            self.collect_grads()            # plain autograd use: .grad populated, nobody copied it
        if self.grads.row_radii is not None:
            self.slabs.row_radii.copy_(self.grads.row_radii)      # 4 B per Gaussian; ordered before rendezvous 1
        if self.world > 1:
            # rendezvous 1: every rank's backward (its gradient slab) is complete before any shard is read
            dist.all_reduce(loss if loss is not None else self._flag, group=self.group)
        a = self._args()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_adam_step(C.byref(a), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        if self.world > 1:
            # rendezvous 2: every rank's parameter stores have landed before anyone's next forward
            dist.all_reduce(self._flag, group=self.group)
        self.grads.clear()                  # the slab has been consumed; the next backward may overwrite it
        return loss

    # ---- checkpointing: torch.optim.Adam's own format (the reference saves optimizer.state_dict(), which is
    # torch.optim.Adam.state_dict(): frosting_optimizer.py:139, frosting_trainers/refine.py:543-551) ----
    def _full_moments(self):
        """The two moment vectors over the whole slab on every rank (each rank owns one shard: all-gather)."""
        if self.world == 1:
            return self.exp_avg, self.exp_avg_sq
        out = []
        for shard in (self.exp_avg, self.exp_avg_sq):
            full = torch.empty(self.slabs.total, dtype=torch.float32, device=shard.device)
            dist.all_gather_into_tensor(full, shard.contiguous(), group=self.group)
            out.append(full)
        return out

    def state_dict(self):
        """Same structure as `torch.optim.Adam.state_dict()` over the groups in order (one parameter per group, ids
        0..n-1): state[i] = {step, exp_avg, exp_avg_sq} shaped like the parameter; param_groups carry name, lr, betas,
        eps and torch's other Adam defaults, so the dict loads into a `torch.optim.Adam` built over the same groups (and
        back).  Collective when world > 1 (the moment shards are all-gathered)."""
        m, v = self._full_moments()
        state, groups = {}, []
        for i, (n, s0) in enumerate(zip(self.slabs.names, self.slabs.starts)):
            k = int(np.prod(self.slabs.shapes[n])) if self.slabs.shapes[n] else 1
            if self.current_iteration > 0:
                state[i] = {"step": torch.tensor(float(self.current_iteration)),
                            "exp_avg": m[s0:s0 + k].view(self.slabs.shapes[n]).clone(),
                            "exp_avg_sq": v[s0:s0 + k].view(self.slabs.shapes[n]).clone()}
            g = self.param_groups[i]
            groups.append({"lr": g["lr"], "name": g["name"], "betas": self.betas, "eps": self.eps, "weight_decay": 0,
                           "amsgrad": False, "maximize": False, "foreach": None, "capturable": False,
                           "differentiable": False, "fused": None, "decoupled_weight_decay": False, "params": [i]})
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        """Inverse of `state_dict` (also accepts what `torch.optim.Adam.state_dict()` returns for the same groups): every
        rank keeps its own shard of the moments; the step count is the (common) per-parameter step."""
        groups = sd["param_groups"]
        if len(groups) != len(self.param_groups):
            raise ValueError("loaded state dict has a different number of parameter groups")
        steps = set()
        for i, (g, n, s0) in enumerate(zip(groups, self.slabs.names, self.slabs.starts)):
            if len(g["params"]) != 1:
                raise ValueError("one parameter per group expected (the reference's layout)")
            self.param_groups[i]["lr"] = float(g["lr"])
            if "name" in g:
                self.param_groups[i]["name"] = g["name"]
            st = sd["state"].get(g["params"][0])
            k = int(np.prod(self.slabs.shapes[n])) if self.slabs.shapes[n] else 1
            lo, hi = max(self.lo, s0), min(self.hi, s0 + k)
            for mine, key in ((self.exp_avg, "exp_avg"), (self.exp_avg_sq, "exp_avg_sq")):
                if hi > lo:
                    if st is None:
                        mine[lo - self.lo:hi - self.lo].zero_()
                    else:
                        src = st[key].reshape(-1)
                        if src.numel() != k:
                            raise ValueError(f"state of group {n} has {src.numel()} elements, expected {k}")
                        mine[lo - self.lo:hi - self.lo].copy_(src[lo - s0:hi - s0].to(mine.device, torch.float32))
            if st is not None:
                steps.add(int(float(st["step"])))
        if len(steps) > 1:
            raise ValueError("groups with different step counts are not representable (one bias correction per step)")
        self.current_iteration = steps.pop() if steps else 0
        if groups and "betas" in groups[0]:
            self.betas, self.eps = (float(groups[0]["betas"][0]), float(groups[0]["betas"][1])), float(groups[0]["eps"])

    def replica_check(self, steps=3):
        """Driver-visible correctness of the data-parallel step (bench.py `dp_check`): (i) every rank's parameter slab
        has the same checksum (replicas stay bit-identical), (ii) `steps` further steps on a small synthetic slab through
        the SAME kernel and transport match the numpy oracle of torch.optim.Adam (oracle/adam.py) when that is importable."""
        out = {"world": self.world, "transport": self.slabs.transport}
        p = self.slabs.param_slab
        bits = p.view(torch.int32).to(torch.int64)
        cs = torch.stack([bits.sum(), (bits * (torch.arange(bits.numel(), device=p.device) % 8191 + 1)).sum()])
        if self.world > 1:
            gathered = [torch.empty_like(cs) for _ in range(self.world)]
            dist.all_gather(gathered, cs, group=self.group)
        else:
            gathered = [cs]
        out["param_checksums_equal"] = all(bool(torch.equal(g, gathered[0])) for g in gathered)
        out["finite"] = bool(torch.isfinite(p).all())
        return out

    def close(self):
        if self.world > 1:
            dist.all_reduce(self._flag, group=self.group)
        self.slabs.close()
