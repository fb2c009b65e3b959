#!/usr/bin/env python
"""The sharded Deallocate (dra_deallocate_batch_global_device) next to the single-context dra_deallocate_batch, on the
records the oracle's Allocate gives for cfg2-shaped batches: 10,000 claims over 125 nodes x 8 GPUs, and 1,000,000 claims
over 10,000 nodes x 8 GPUs (80,000 GPUs).  Nodes are split evenly over the ranks.

Every context loads the inventory as that Allocate left it, so dra_reset_inventory (an untimed device-to-device copy on the
context's stream) restores the same starting state before each timed call and no record is released twice.  Before
timing, one call on every rank must leave each rank's own GPU range equal to the CPU oracle's spec §9 state and every other
GPU as loaded, and dra_deallocate_batch on one context must leave the oracle's state.  The sharded call is timed with CUDA
events on each rank's stream around the call: the max over ranks of the mean over --steps calls.  dra_deallocate_batch
takes host buffers and synchronises, so it is timed with the host clock around the call (its staging copy into pinned
memory, both transfers and the kernel).  Prints one JSON line with the card name and power limit.

  python profiles/shard_dealloc.py [--steps K]            world 1: one context serving every node
  python profiles/shard_dealloc.py --local-world K        K contexts of one process on GPU 0 (dra_comm_init_local)
"""
import argparse, importlib, json, os, subprocess, sys, time
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("k8s-dra-driver_b200")
from oracle import oracle as O
api, R = pkg.api, pkg.records

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=100)
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--local-world", type=int, default=1)
args = ap.parse_args()
world = args.local_world
dev = torch.device("cuda", 0)

res, fails = {}, 0
for key, n_claim, n_node in (("cfg2_10k_claims", 10_000, 125), ("claims_1m_gpus_80000", 1_000_000, 10_000)):
    w = pkg.synth.cfg2(n_claim, n_node)
    n_out = int(w.n_out)
    ref, allocated = O.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, n_out)
    want = O.deallocate(allocated, w.claims, ref, w.out_off, n_node=n_node)
    assert (ref["status"] == R.ST_OK).any() and want.tobytes() != allocated.tobytes()
    bounds = [n_node * r // world for r in range(world)] + [n_node]
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    ctxs = [api.Context(device=0, stream=s.cuda_stream) for s in streams]
    for r, c in enumerate(ctxs):
        c.comm_init_local(r, world)
        c.set_table(w.table); c.set_inventory(allocated, w.node_off); c.set_shard_map(bounds, stray_rank=0)
    single = api.Context(device=0)
    single.set_table(w.table); single.set_inventory(allocated, w.node_off)
    d_c = torch.from_numpy(w.claims.view(np.uint8).copy()).to(dev)
    d_o = torch.from_numpy(w.out_off.view(np.uint8).copy()).to(dev) if w.out_off is not None else None
    d_r = torch.from_numpy(ref[:n_out].view(np.uint8).copy()).to(dev)
    o_ptr = d_o.data_ptr() if d_o is not None else None
    torch.cuda.synchronize()

    # parity first
    for c in ctxs:
        c.deallocate_global_device(d_c.data_ptr(), n_claim, o_ptr, d_r.data_ptr(), n_out)
    ok = True
    for r, c in enumerate(ctxs):
        c.sync()
        inv = c.get_inventory()
        g0, g1 = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        ok = ok and inv[g0:g1].tobytes() == want[g0:g1].tobytes()
        ok = ok and inv[:g0].tobytes() == allocated[:g0].tobytes() and inv[g1:].tobytes() == allocated[g1:].tobytes()
    single.deallocate(w.claims, ref[:n_out], w.out_off)
    ok = ok and single.get_inventory().tobytes() == want.tobytes()
    if not ok:
        fails += 1
        print(f"{key}: MISMATCH against the oracle; not timed", file=sys.stderr)
        continue                                       # a wrong answer is not timed
    # the sharded call: events on each rank's stream, every rank's call enqueued before any waits
    evs = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
           for _ in ctxs]
    for i in range(args.warmup + args.steps):
        for c in ctxs:
            c.reset_inventory()
        for r, c in enumerate(ctxs):
            if i >= args.warmup:
                evs[r][i - args.warmup][0].record(streams[r])
            c.deallocate_global_device(d_c.data_ptr(), n_claim, o_ptr, d_r.data_ptr(), n_out)
            if i >= args.warmup:
                evs[r][i - args.warmup][1].record(streams[r])
    for c in ctxs:
        c.sync()
    us = max(sum(a.elapsed_time(b) for a, b in evs[r]) / args.steps * 1e3 for r in range(world))
    # the per-rank call on one context: host clock around the call
    host = []
    for i in range(args.warmup + args.steps):
        single.reset_inventory()
        single.sync()
        t0 = time.perf_counter()
        single.deallocate(w.claims, ref[:n_out], w.out_off)
        if i >= args.warmup:
            host.append(time.perf_counter() - t0)
    res[key] = {"claims": n_claim, "records": n_out, "gpus": int(w.n_gpu),
                "bytes_read_per_rank": n_claim * (16 + (4 if w.out_off is not None else 0)) + n_out * 8,
                "global_device_us_per_call": round(us, 2),
                "deallocate_batch_host_us_per_call": round(float(np.mean(host)) * 1e6, 2)}
    for c in ctxs:
        c.close()
    single.close()
q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip()
print(json.dumps({"call": "dra_deallocate_batch_global_device", "ranks": world,
                  "layout": "one context" if world == 1 else "contexts of one process on one GPU",
                  "gpu": q, "parity": "every rank's range bit-exact vs oracle, nothing written outside it" if not fails
                  else "MISMATCH", **res}))
sys.exit(1 if fails else 0)
