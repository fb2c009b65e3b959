#!/usr/bin/env python
"""The inventory sync of a sharded world (dra_shard_sync_inventory_device) at cfg3's 8,000 GPUs (1,000 nodes x 8, 128 KB of
records) and at 80,000 GPUs (10,000 nodes x 8, 1.28 MB).  Nodes are split evenly over the ranks.  Before timing, a sharded
Allocate and a sync must leave every rank's whole inventory equal to the CPU oracle's.  Device time per call: CUDA events on
each rank's stream around the call, after a device-side rendezvous of the ranks (dra_peer_rendezvous_device) so that no
rank's time includes a peer's late start; the max over ranks of the mean over --steps calls.  Prints one JSON line with the
card name and power limit.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 profiles/shard_sync.py [--steps K]
      one process per GPU (N >= 2), peers mapped with IPC handles
  python profiles/shard_sync.py --local-world K
      K contexts of one process on GPU 0 (dra_comm_init_local / dra_peer_import_local): the protocol without NVLink
"""
import argparse, importlib, json, os, subprocess, sys
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("k8s-dra-driver_b200")
from oracle import oracle as O

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=200)
ap.add_argument("--warmup", type=int, default=20)
ap.add_argument("--local-world", type=int, default=0)
args = ap.parse_args()

if args.local_world:
    world, rank, local, dist = args.local_world, 0, 0, None
    ranks = list(range(world))
else:
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    ranks = [rank]
if world < 2:
    sys.exit("the sync enqueues nothing at world 1: run it with N >= 2 processes or --local-world K >= 2")
dev = torch.device("cuda", local)
streams = {r: torch.cuda.Stream(device=dev) for r in ranks}


def setup(w, bounds):
    ctxs = {r: pkg.api.Context(device=local, stream=streams[r].cuda_stream) for r in ranks}
    for r, c in ctxs.items():
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
    if dist is None:
        for r, c in ctxs.items():
            c.comm_init_local(r, world); c.set_shard_map(bounds, stray_rank=0); c.shard_export(w.n_out, 0, want_handle=False)
        for c in ctxs.values():
            c.peer_import_local([ctxs[r] for r in ranks])
    else:
        c = ctxs[rank]
        uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        c.comm_init(uid[0], rank, world); c.set_shard_map(bounds, stray_rank=0)
        hs = [None] * world
        dist.all_gather_object(hs, c.shard_export(w.n_out))
        c.peer_import(hs)
    return ctxs


def all_ok(ok):
    if dist is None:
        return ok
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    return int(t.item()) == 0


res, fails = {}, 0
for key, n_node in (("cfg3_8000_gpus", 1000), ("gpus_80000", 10_000)):
    w = pkg.synth.cfg3(20_000, n_node)
    bounds = [n_node * r // world for r in range(world)] + [n_node]
    ctxs = setup(w, bounds)
    # parity first: a sharded Allocate makes the copies diverge, the sync makes every one the oracle's state
    ref, state = O.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    d_c = torch.from_numpy(w.claims.view(np.uint8).copy()).to(dev)          # cfg3: one slot per claim, no out_off
    torch.cuda.synchronize()
    for c in ctxs.values():
        c.allocate_global_device(d_c.data_ptr(), w.n_claim, None, w.n_out, 0)
    for c in ctxs.values():
        c.shard_sync_inventory_device()
    for c in ctxs.values():
        c.sync()
    if not all_ok(all(c.get_inventory().tobytes() == state.tobytes() for c in ctxs.values())):
        fails += 1
        continue                                       # a wrong answer is not timed
    evs = {r: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
           for r in ranks}
    for i in range(args.warmup + args.steps):
        for c in ctxs.values():
            c.peer_rendezvous()
        for r, c in ctxs.items():
            if i >= args.warmup:
                evs[r][i - args.warmup][0].record(streams[r])
            c.shard_sync_inventory_device()
            if i >= args.warmup:
                evs[r][i - args.warmup][1].record(streams[r])
    for c in ctxs.values():
        c.sync()
    us = max(sum(a.elapsed_time(b) for a, b in evs[r]) / args.steps * 1e3 for r in ranks)
    if dist is not None:
        t = torch.tensor([us], dtype=torch.float64, device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); us = float(t.item())
    res[key] = {"gpus": w.n_gpu, "record_bytes": w.n_gpu * 16, "us_per_call": round(us, 2)}
    for c in ctxs.values():
        c.close()
if rank == 0:
    q = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"call": "dra_shard_sync_inventory_device", "ranks": world,
                      "layout": "contexts of one process on one GPU" if dist is None else "one process per GPU",
                      "gpu": q, "parity": "every rank's inventory bit-exact vs oracle" if not fails else "MISMATCH", **res}))
if dist is not None:
    dist.destroy_process_group()
sys.exit(1 if fails else 0)
