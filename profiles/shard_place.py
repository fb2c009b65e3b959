#!/usr/bin/env python
"""Sharded place pods (dra_place_pods_batch_global_device) against dra_place_pods_batch on the same input.  Workloads:
  s13_dense / s13_random8   spec §13's workload: synth.pods, 20,000 pods over 64 nodes, the dense form and 8 random
                            candidates per pod (some naming no node)
  wide_random8              10,000 nodes with 8 random candidates for each of 20,000 pods: more nodes than one GPU's
                            resident warps of k_pods_place<4>, so each warp cycles over several nodes
Nodes are split evenly over the ranks.  Every call starts from the pristine inventory (DRA_F_FRESH_INVENTORY), first-fit
and exhaustive.  Before timing, every rank's table, pod_node and own inventory range are checked against the CPU oracle
(tests/place_oracle.py).  Device time per call: CUDA events on each rank's stream around the call, after a device-side
rendezvous of the ranks; the max over ranks of the mean over --steps calls (it includes the all-gather).  Rank 0 then times
dra_place_pods_batch on one context holding the whole inventory (events on its stream, so the time includes its own
copies in and out).  Prints one JSON line with the card name and power limit.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 profiles/shard_place.py [--steps K]
      one process per GPU, peers mapped with IPC handles
  python profiles/shard_place.py --local-world K
      K contexts of one process on GPU 0 (dra_comm_init_local / dra_peer_import_local): the protocol without NVLink
"""
import argparse, importlib, json, os, subprocess, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("k8s-dra-driver_b200")
import place_oracle as P

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--local-world", type=int, default=0)
ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
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
dev = torch.device("cuda", local)
streams = {r: torch.cuda.Stream(device=dev) for r in ranks}
A = pkg.api


def setup(w, bounds, n_pod):
    ctxs = {r: A.Context(device=local, stream=streams[r].cuda_stream) for r in ranks}
    for r, c in ctxs.items():
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
    if dist is None:
        for r, c in ctxs.items():
            c.comm_init_local(r, world); c.set_shard_map(bounds, stray_rank=0)
            if world > 1:
                c.set_shard_place(n_pod); c.shard_export(w.n_claim, 0, want_handle=False)
        if world > 1:
            for c in ctxs.values():
                c.peer_import_local([ctxs[r] for r in ranks])
    else:
        c = ctxs[rank]
        uid = [A.Context.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        c.comm_init(uid[0], rank, world); c.set_shard_map(bounds, stray_rank=0)
        if world > 1:
            c.set_shard_place(n_pod)
            hs = [None] * world
            dist.all_gather_object(hs, c.shard_export(w.n_claim))
            c.peer_import(hs)
    return ctxs


def all_ok(ok):
    if dist is None:
        return ok
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    return int(t.item()) == 0


def dv(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev)


rng = np.random.default_rng(11)
work = {}
w13, po13 = pkg.synth.pods(20_000, 64, 3)
n13 = len(po13) - 1
work["s13_dense"] = (w13, po13, None, None)
work["s13_random8"] = (w13, po13, rng.integers(0, 66, n13 * 8).astype(np.uint32), (np.arange(n13 + 1) * 8).astype(np.uint32))
ww, pow_ = pkg.synth.pods(20_000, 10_000, 5)
nw = len(pow_) - 1
work["wide_random8"] = (ww, pow_, rng.integers(0, 10_002, nw * 8).astype(np.uint32), (np.arange(nw + 1) * 8).astype(np.uint32))
only = [x for x in args.only.split(",") if x]

res, fails = {}, 0
for name, (w, pod_off, cn, co) in work.items():
    if only and name not in only:
        continue
    n_pod = len(pod_off) - 1
    bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
    ctxs = setup(w, bounds, n_pod)
    d_c, d_p = dv(w.claims), dv(pod_off)
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    n_pair = int(co[-1]) if co is not None else 0
    pn = {r: torch.zeros(n_pod * 4, dtype=torch.uint8, device=dev) for r in ranks}
    torch.cuda.synchronize()
    for key, fl in (("first_fit", A.F_FRESH_INVENTORY), ("exhaustive", A.F_FRESH_INVENTORY | A.F_EXHAUSTIVE)):
        def call(r, c):
            c.place_pods_global_device(d_c.data_ptr(), w.n_claim, d_p.data_ptr(), n_pod,
                                       d_n.data_ptr() if d_n is not None else None, d_o.data_ptr() if d_o is not None else None,
                                       n_pair, None, w.n_claim, pn[r].data_ptr(), fl)
        print(f"{name} {key}: checking against the oracle", file=sys.stderr, flush=True)
        for r, c in ctxs.items():
            call(r, c)
        for c in ctxs.values():
            c.sync()
        ref, ref_node, ref_inv = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, None, w.n_claim,
                                              P.F_EXHAUSTIVE if fl & A.F_EXHAUSTIVE else 0)
        ok = True
        for r, c in ctxs.items():
            g0, g1 = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
            got = c.gather_read(np.zeros(w.n_claim, dtype=pkg.records.OUT_DTYPE))
            ok = ok and got.tobytes() == ref.tobytes() and c.get_inventory()[g0:g1].tobytes() == ref_inv[g0:g1].tobytes() \
                and pn[r].cpu().numpy().view(np.uint32).tobytes() == ref_node.tobytes()
        if not all_ok(ok):
            fails += 1
            continue                                   # a wrong answer is not timed
        evs = {r: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
               for r in ranks}
        for i in range(args.warmup + args.steps):
            if world > 1:
                for c in ctxs.values():
                    c.peer_rendezvous()
            for r, c in ctxs.items():
                if i >= args.warmup:
                    evs[r][i - args.warmup][0].record(streams[r])
                call(r, c)
                if i >= args.warmup:
                    evs[r][i - args.warmup][1].record(streams[r])
        for c in ctxs.values():
            c.sync()
        us = max(sum(a.elapsed_time(b) for a, b in evs[r]) / args.steps * 1e3 for r in ranks)
        if dist is not None:
            t = torch.tensor([us], dtype=torch.float64, device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); us = float(t.item())
        res.setdefault(name, {})[key] = {"us_per_call": round(us, 1), "placed": int((ref_node != 0xFFFFFFFF).sum())}
        if rank == 0:                                  # the single-inventory call on the same input, whole inventory
            with A.Context(device=local, stream=streams[ranks[0]].cuda_stream) as single:
                single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
                out, node = single.place_pods(w.claims, pod_off, cn, co, None, w.n_claim, fl)
                if out.tobytes() != ref.tobytes() or node.tobytes() != ref_node.tobytes():
                    fails += 1
                else:
                    s = streams[ranks[0]]
                    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
                    for a, b in ev:
                        a.record(s); single.place_pods(w.claims, pod_off, cn, co, None, w.n_claim, fl); b.record(s)
                    s.synchronize()
                    res[name][key]["single_inventory_us_per_call"] = round(sum(a.elapsed_time(b) for a, b in ev) / args.steps * 1e3, 1)
        if dist is not None:
            dist.barrier()
    for c in ctxs.values():
        c.close()
if rank == 0:
    q = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"call": "dra_place_pods_batch_global_device", "ranks": world,
                      "layout": "contexts of one process on one GPU" if dist is None else "one process per GPU",
                      "gpu": q, "parity": "every rank's table, pod_node and own range bit-exact vs oracle" if not fails
                      else "MISMATCH", **res}))
if dist is not None:
    dist.destroy_process_group()
sys.exit(1 if fails else 0)
