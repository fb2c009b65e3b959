#!/usr/bin/env python
"""Sharded UnsuitableNodes (dra_unsuitable_batch_global_device) at N GPUs: 10,000 pods x every node of the global cfg2
inventory (N x 125 nodes, dense) against a half-full inventory, first-fit and exhaustive.  One process per GPU (torchrun),
gather buffers mapped with IPC handles.  Before timing, every rank's bitmap is checked against the CPU oracle on the first
500 pods.  Device time per call: CUDA events on the launch stream, L2 flushed before each call, max over ranks; it
includes the bit exchange.  Rank 0 prints one JSON line with the card name and power limit.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 profiles/shard_unsuitable.py [--steps K]
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
N_POD, NODES_PER_RANK, N_CHECK = 10_000, 125, 500

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
os.environ.setdefault("NCCL_DEBUG", "WARN")
torch.cuda.set_device(local)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

w = pkg.synth.cfg2(10_000 * world, NODES_PER_RANK * world, 8)
_, inv = O.allocate(w.gpus, w.node_off, w.table, w.claims[: 4000 * world], threads=8)      # half full
ctx = pkg.api.Context(device=local, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(inv, w.node_off)
uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], rank, world)
ctx.set_shard_map([w.n_node * r // world for r in range(world)] + [w.n_node], stray_rank=0)
n_pair = N_POD * w.n_node
if world > 1:
    ctx.set_shard_pairs(n_pair)
    hs = [None] * world
    dist.all_gather_object(hs, ctx.shard_export(w.n_out))
    ctx.peer_import(hs)

pods = w.claims[:N_POD].copy()
pod_off = np.arange(N_POD + 1, dtype=np.uint32)
d_c = torch.from_numpy(pods.view(np.uint8).copy()).to(dev)
d_po = torch.from_numpy(pod_off.view(np.uint8).copy()).to(dev)
d_bits = torch.zeros((n_pair + 7) // 8, dtype=torch.uint8, device=dev)
cn = np.tile(np.arange(w.n_node, dtype=np.uint32), N_CHECK)
co = (np.arange(N_CHECK + 1, dtype=np.uint64) * w.n_node).astype(np.uint32)
res, fails = {}, 0
for key, fl, ofl in (("first_fit", 0, 0), ("exhaustive", pkg.api.F_EXHAUSTIVE, O.F_EXHAUSTIVE)):
    def call():
        ctx.unsuitable_global_device(d_c.data_ptr(), N_POD, d_po.data_ptr(), N_POD, None, None, n_pair, d_bits.data_ptr(), fl)
    call(); ctx.sync()
    bits = d_bits.cpu().numpy()
    ref = O.unsuitable(inv, w.node_off, w.table, pods[:N_CHECK], pod_off[: N_CHECK + 1], cn, co, flags=ofl)
    ok = bits[: len(ref) - 1].tobytes() == ref[: len(ref) - 1].tobytes()
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    if int(t.item()):
        fails += 1
        continue                                       # a wrong answer is not timed
    for _ in range(args.warmup):
        flush.fill_(1); call()
    ctx.sync(); dist.barrier()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for a, b in evs:
        flush.fill_(1)
        a.record(stream); call(); b.record(stream)
    ctx.sync(); dist.barrier()
    ms = torch.tensor([sum(a.elapsed_time(b) for a, b in evs) / args.steps], dtype=torch.float64, device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    res[key] = {"us_per_call": float(ms.item()) * 1e3, "pairs_per_s": n_pair / (float(ms.item()) * 1e-3),
                "suitable_pairs": int(np.unpackbits(bits).sum())}
if rank == 0:
    q = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"call": "dra_unsuitable_batch_global_device", "n_gpus": world, "pods": N_POD, "nodes": w.n_node,
                      "pairs": n_pair, "gpu": q, "parity": f"first {N_CHECK} pods bit-exact vs oracle on every rank"
                      if not fails else "MISMATCH", **res}))
ctx.close()
dist.destroy_process_group()
sys.exit(1 if fails else 0)
