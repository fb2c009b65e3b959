#!/usr/bin/env python
"""Sharded place pods with reasons (dra_place_pods_why_batch_global_device) against the sharded place pods alone
(dra_place_pods_batch_global_device) on the same world, and against dra_place_pods_why_batch on one context holding the
whole inventory.  Workloads: profiles/shard_place.py's (s13_dense, s13_random8: synth.pods, 20,000 pods over 64 nodes;
wide_random8: 20,000 pods over 10,000 nodes, 8 random candidates each).  K contexts of one process on GPU 0 for each K of
--worlds (dra_comm_init_local / dra_peer_import_local), nodes split evenly, every call from the pristine inventory
(DRA_F_FRESH_INVENTORY), first-fit and exhaustive.

Before timing: every rank's table, pod_node and own inventory range against the CPU oracle (tests/place_oracle.py), and
every rank's four reason outputs against dra_place_pods_why_batch on the whole inventory (the reasons oracle,
tests/place_why_oracle.py, is too slow in Python at these sizes; the single-inventory call is held to it by
tests/test_gpu_place_why.py).  Device time per call: CUDA events on each rank's stream around the call, after a
device-side rendezvous; the max over ranks of the mean over --steps calls.  Prints one JSON line with the card name and
power limit.

  python profiles/shard_place_why.py [--worlds 1,2,4] [--steps K] [--only s13_random8,...]
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
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--worlds", default="1,2,4")
ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
args = ap.parse_args()
A = pkg.api
dev = torch.device("cuda", 0)
WHY_N = A.WHY_N


def dv(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(dev) if a.nbytes else torch.zeros(16, dtype=torch.uint8, device=dev)


def setup(w, world, bounds, n_pod, n_why, streams):
    ctxs = [A.Context(device=0, stream=streams[r].cuda_stream) for r in range(world)]
    for r, c in enumerate(ctxs):
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        c.comm_init_local(r, world); c.set_shard_map(bounds, stray_rank=0)
        if world > 1:
            c.set_shard_place(n_pod); c.set_shard_why(n_why); c.shard_export(w.n_claim, 0, want_handle=False)
    if world > 1:
        for c in ctxs:
            c.peer_import_local(ctxs)
    return ctxs


def timed(ctxs, streams, call):
    evs = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
           for _ in ctxs]
    for i in range(args.warmup + args.steps):
        if len(ctxs) > 1:
            for c in ctxs:
                c.peer_rendezvous()
        for r, c in enumerate(ctxs):
            if i >= args.warmup:
                evs[r][i - args.warmup][0].record(streams[r])
            call(r, c)
            if i >= args.warmup:
                evs[r][i - args.warmup][1].record(streams[r])
    for c in ctxs:
        c.sync()
    return round(max(sum(a.elapsed_time(b) for a, b in e) / args.steps * 1e3 for e in evs), 1)


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
    n_pair = int(co[-1]) if co is not None else 0
    n_why = n_pod * w.n_node if co is None else n_pair
    d_c, d_p = dv(w.claims), dv(pod_off)
    d_n, d_o = (dv(cn), dv(co)) if co is not None else (None, None)
    for key, fl in (("first_fit", A.F_FRESH_INVENTORY), ("exhaustive", A.F_FRESH_INVENTORY | A.F_EXHAUSTIVE)):
        ref, ref_node, ref_inv = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, None, w.n_claim,
                                              P.F_EXHAUSTIVE if fl & A.F_EXHAUSTIVE else 0)
        s0 = torch.cuda.Stream(device=dev)
        with A.Context(device=0, stream=s0.cuda_stream) as single:
            single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
            one = single.place_pods_why(w.claims, pod_off, cn, co, None, w.n_claim, fl)
            if one[0].tobytes() != ref.tobytes() or one[1].tobytes() != ref_node.tobytes():
                fails += 1
                continue
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            single.place_pods_why(w.claims, pod_off, cn, co, None, w.n_claim, fl)
            for a, b in ev:
                a.record(s0); single.place_pods_why(w.claims, pod_off, cn, co, None, w.n_claim, fl); b.record(s0)
            s0.synchronize()
            entry = {"placed": int((ref_node != 0xFFFFFFFF).sum()), "pairs": n_why,
                     "single_why_us_per_call": round(sum(a.elapsed_time(b) for a, b in ev) / args.steps * 1e3, 1)}
        for world in [int(x) for x in args.worlds.split(",")]:
            print(f"{name} {key} K={world}: checking", file=sys.stderr, flush=True)
            bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
            streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
            ctxs = setup(w, world, bounds, n_pod, n_why, streams)
            pn = [torch.zeros(n_pod * 4, dtype=torch.uint8, device=dev) for _ in range(world)]
            outs = [[torch.zeros(s, dtype=torch.uint8, device=dev) for s in (n_why, n_why * 4, n_pod * WHY_N * 4, w.n_claim * 4)]
                    for _ in range(world)]
            torch.cuda.synchronize()

            def why(r, c):
                c.place_pods_why_global_device(d_c.data_ptr(), w.n_claim, d_p.data_ptr(), n_pod,
                                               None if d_n is None else d_n.data_ptr(), None if d_o is None else d_o.data_ptr(),
                                               n_pair, None, w.n_claim, pn[r].data_ptr(), *[o.data_ptr() for o in outs[r]],
                                               flags=fl)

            def place(r, c):
                c.place_pods_global_device(d_c.data_ptr(), w.n_claim, d_p.data_ptr(), n_pod,
                                           None if d_n is None else d_n.data_ptr(), None if d_o is None else d_o.data_ptr(),
                                           n_pair, None, w.n_claim, pn[r].data_ptr(), fl)

            for r, c in enumerate(ctxs):
                why(r, c)
            for c in ctxs:
                c.sync()
            ok = True
            for r, c in enumerate(ctxs):
                g0, g1 = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
                got = [o.cpu().numpy().view(d) for o, d in zip(outs[r], (np.uint8, np.uint32, np.uint32, np.uint32))]
                ok = ok and c.gather_read(np.zeros(w.n_claim, dtype=pkg.records.OUT_DTYPE)).tobytes() == ref.tobytes() \
                    and c.get_inventory()[g0:g1].tobytes() == ref_inv[g0:g1].tobytes() \
                    and pn[r].cpu().numpy().view(np.uint32).tobytes() == ref_node.tobytes() \
                    and all(x.tobytes() == np.ascontiguousarray(y, x.dtype).tobytes() for x, y in zip(got, one[2:]))
            if not ok:
                fails += 1
            else:
                entry[f"K{world}"] = {"why_us_per_call": timed(ctxs, streams, why), "place_us_per_call": timed(ctxs, streams, place)}
            for c in ctxs:
                c.close()
        res.setdefault(name, {})[key] = entry
q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip()
print(json.dumps({"call": "dra_place_pods_why_batch_global_device", "layout": "contexts of one process on one GPU",
                  "gpu": q, "parity": "every rank's outputs bit-exact" if not fails else "MISMATCH", **res}))
sys.exit(1 if fails else 0)
