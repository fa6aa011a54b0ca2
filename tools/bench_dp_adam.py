"""Device time of the data-parallel Adam step alone (row f3), under torchrun.
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/bench_dp_adam.py [P]
Prints, per world size, the max over ranks (which meet before each timed region) of:
- the peer-memory reduce + Adam + publish kernel alone: ms per launch, CUDA events around 20 launches, and its NVLink
  payload rate per GPU and direction and its local HBM rate;
- `FrostingAdam.step()` with dense gradient rows and with sparse ones (runs of 4096 rows, one run in ten rendered, as
  a frame's visible Gaussians cluster), alternating, fresh gradients before each: medians of 8 steps after 2 warm-up
  rounds."""
import os
import sys
import ctypes as C

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frosting_b200 import optim, _lib   # noqa: E402
from tools import timing                # noqa: E402


def main():
    P = int(sys.argv[1]) if len(sys.argv) > 1 else 2_000_000
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    shapes = {"bary_logits": (P, 6), "sh_dc": (P, 1, 3), "sh_rest": (P, 15, 3), "opacity_logits": (P,),
              "log_scales": (P, 3), "quats": (P, 4)}
    g = torch.Generator().manual_seed(1)
    params = {k: torch.randn(s, generator=g).to(dev) for k, s in shapes.items()}
    opt = optim.FrostingAdam.for_frosting(params)
    n = opt.slabs.total
    stream = torch.cuda.current_stream(dev)
    L = _lib.lib()
    radii = ((torch.arange(P, device=dev) // 4096 + rank) % 10 == 0).int() * 5

    def fresh_grads():           # every group written, as a backward leaves them; ranks meet before the window opens
        for k in shapes:
            opt.grads[k].normal_()
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()

    def launch():
        opt.current_iteration += 1
        a = opt._args()
        _lib.check(L.fb200_adam_step(C.byref(a), C.c_void_p(stream.cuda_stream)))

    def sparse_step():           # the rows are declared as frosting_render's backward does: host bookkeeping only
        opt.grads.rows_from(radii, list(shapes))
        opt.step()

    iters = 20
    kernel = timing.alternate({"launches": lambda: [launch() for _ in range(iters)]}, 1, 1, before=fresh_grads)[0]
    step = timing.alternate({"dense": opt.step, "sparse": sparse_step}, 8, 2, before=fresh_grads)[0]
    t = torch.tensor([kernel["launches"]["median_ms"] / iters, step["dense"]["median_ms"], step["sparse"]["median_ms"]],
                     device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, dense, sparse = t.tolist()
    shard = (opt.hi - opt.lo) * 4
    remote = shard * (world - 1)                 # bytes in (gradients) = bytes out (parameters), per GPU
    hbm = shard * (1 + 3 + 3) + 2 * remote       # own grad + m,v,p reads + m,v,p writes + what the peers read / write here
    if rank == 0:
        print(f"world {world} [{opt.slabs.transport}]: {n / 1e6:.1f} M parameters, {ms:.3f} ms per step; NVLink {remote / 1e6:.0f} MB each way per GPU "
              f"-> {remote / ms / 1e6:.0f} GB/s per direction; local HBM traffic {hbm / 1e6:.0f} MB -> {hbm / ms / 1e6:.0f} GB/s")
        print(f"world {world} [{opt.slabs.transport}]: FrostingAdam.step() dense {dense:.3f} ms, sparse rows {sparse:.3f} ms")
    if world > 1:
        dist.barrier()
    opt.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
