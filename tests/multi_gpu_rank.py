"""The rank setup every torchrun multi-GPU check (tests/multi_gpu_*check.py) shares: one process per GPU, NCCL for the host
collectives, the sharded world's peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  Each check is
reduced over the ranks and printed by rank 0; the run ends with "ALL OK" or "N FAILURES" and the matching exit code.  Not
collected by pytest: tests/test_gpu_multi_rank.py launches the scripts."""
import importlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("k8s-dra-driver_b200")

rank = world = dev = None
fails = 0


def start():
    """The NCCL init of this rank; returns (rank, world, device, stream), the stream made torch's current one."""
    global rank, world, dev
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    return rank, world, dev, stream


def join(ctx, bounds, stray_rank, n_out, **sizes):
    """ctx joins the world: communicator, shard map, one dra_set_shard_<name>(*args) per keyword (pairs=(n,), ...), the
    export of an n_out-record table and the import of every rank's handle."""
    uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(uid[0], rank, world)
    ctx.set_shard_map(bounds, stray_rank=stray_rank)
    for name, args in sizes.items():
        getattr(ctx, "set_shard_" + name)(*args)
    hs = [None] * world
    dist.all_gather_object(hs, ctx.shard_export(n_out))
    ctx.peer_import(hs)


def dv(a):
    """a's bytes on this rank's device; 16 zero bytes for an empty array, so the pointer is never null."""
    a = np.ascontiguousarray(a)
    if a.nbytes == 0:
        return torch.zeros(16, dtype=torch.uint8, device=dev)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(dev)


def report(what, ok, detail=None):
    """One check: OK only if it held on every rank.  Rank 0 prints it; a failure is counted.  Returns whether it held."""
    global fails
    t = torch.tensor([0 if ok else 1], device=dev)
    dist.all_reduce(t)
    bad = int(t.item()) != 0
    fails += bad
    if rank == 0:
        print(f"{what}: {'MISMATCH' if bad else 'OK'}" + ("" if detail is None else f" ({detail})"))
    return not bad


def finish(ctxs=()):
    """Close the contexts once every rank is done, print the verdict on rank 0 and exit with it.  Every rank counted every
    failed check (report() reduces each one), so the count is the largest rank's, not the sum."""
    dist.barrier()
    for c in ctxs:
        c.close()
    t = torch.tensor([fails], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print("ALL OK" if int(t.item()) == 0 else f"{int(t.item())} FAILURES")
    dist.destroy_process_group()
    sys.exit(1 if int(t.item()) else 0)
