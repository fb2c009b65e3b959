#!/usr/bin/env python
"""Sharded pods Allocate (dra_allocate_pods_batch_global_device) at N GPUs: synth.pods scaled by N (N x 20,000 pods of 1-5
MIG claims over N x 64 pre-fragmented nodes), first-fit and exhaustive, each call from the pristine inventory
(DRA_F_FRESH_INVENTORY, so every step does the same work).  One process per GPU (torchrun), gather buffers mapped with IPC
handles.  Before timing, every rank's whole table and own inventory range are checked against the CPU oracle.  Device time
per call: CUDA events on the launch stream, L2 flushed before each call, max over ranks; it includes the all-gather.
Rank 0 then times dra_allocate_pods_batch, the single-inventory call, on the same pods and the whole inventory (events on
the same stream, so its time includes its host-to-device and device-to-host copies).  Rank 0 prints one JSON line with
the card name and power limit.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 profiles/shard_pods.py [--steps K]
"""
import argparse, importlib, json, os, subprocess, sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("k8s-dra-driver_b200")
from oracle import oracle as O

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
args = ap.parse_args()
PODS_PER_RANK, NODES_PER_RANK = 20_000, 64

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
os.environ.setdefault("NCCL_DEBUG", "WARN")
torch.cuda.set_device(local)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

w, pod_off = pkg.synth.pods(PODS_PER_RANK * world, NODES_PER_RANK * world, 3)
n_pod = len(pod_off) - 1
bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
ctx = pkg.api.Context(device=local, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], rank, world)
ctx.set_shard_map(bounds, stray_rank=0)
if world > 1:
    hs = [None] * world
    dist.all_gather_object(hs, ctx.shard_export(w.n_claim))
    ctx.peer_import(hs)

d_c = torch.from_numpy(w.claims.view(np.uint8).copy()).to(dev)
d_po = torch.from_numpy(pod_off.view(np.uint8).copy()).to(dev)
torch.cuda.synchronize()


def timed(call):
    for _ in range(args.warmup):
        flush.fill_(1); call()
    ctx.sync()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for a, b in evs:
        flush.fill_(1)
        a.record(stream); call(); b.record(stream)
    ctx.sync()
    return sum(a.elapsed_time(b) for a, b in evs) / args.steps


res, fails = {}, 0
for key, fl, ofl in (("first_fit", 0, 0), ("exhaustive", pkg.api.F_EXHAUSTIVE, O.F_EXHAUSTIVE)):
    fl |= pkg.api.F_FRESH_INVENTORY

    def call():
        ctx.allocate_pods_global_device(d_c.data_ptr(), w.n_claim, d_po.data_ptr(), n_pod, None, w.n_claim, fl)
    call(); ctx.sync()
    got = ctx.gather_read(np.zeros(w.n_claim, dtype=pkg.records.OUT_DTYPE))
    ref, ref_inv = O.allocate_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, flags=ofl)
    ok = got.tobytes() == ref.tobytes() and ctx.get_inventory()[g0:g1].tobytes() == ref_inv[g0:g1].tobytes()
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    if int(t.item()):
        fails += 1
        continue                                       # a wrong answer is not timed
    dist.barrier()
    ms = torch.tensor([timed(call)], dtype=torch.float64, device=dev)
    dist.barrier()
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    res[key] = {"us_per_call": float(ms.item()) * 1e3, "ok_slots": int((ref["status"] == 0).sum())}
    if rank == 0:                                      # the single-inventory call on the same pods, whole inventory
        single = ctx.allocate_pods(w.claims, pod_off, None, w.n_claim, fl)
        if single.tobytes() != ref.tobytes():
            fails += 1
        else:
            res[key]["single_inventory_us_per_call"] = timed(lambda: ctx.allocate_pods(w.claims, pod_off, None, w.n_claim, fl)) * 1e3
    dist.barrier()
if rank == 0:
    q = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"call": "dra_allocate_pods_batch_global_device", "n_gpus": world, "pods": n_pod, "claims": w.n_claim,
                      "nodes": w.n_node, "gpu": q, "parity": "every rank's table and own range bit-exact vs oracle"
                      if not fails else "MISMATCH", **res}))
ctx.close()
dist.destroy_process_group()
sys.exit(1 if fails else 0)
