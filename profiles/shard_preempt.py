#!/usr/bin/env python
"""Sharded preemption (dra_preempt_batch_global_device, spec §14 "Sharded form") next to what it replaces.  The two
workloads of profiles/preempt.py (DESIGN §4, "Preemption"): the cfg2-sized fragmented MIG world and the SHARED-heavy
world, 1,000 pending pods, dense (125,000 pairs) and 16 random candidates per pod, flags 0 and DRA_F_EXHAUSTIVE.  Every
rank's six outputs are checked against the CPU oracle before anything is timed.  Three times per case, median of --steps
calls after --warmup:
  sharded     the sharded call, CUDA events on each rank's stream after dra_peer_rendezvous_device, max over ranks
              (device-resident inputs and outputs; the partials' exchange included)
  single      dra_preempt_batch on one context (host buffers, as profiles/preempt.py times it)
  sync+single the workaround the sharded call replaces: dra_shard_sync_inventory_device on every rank (events on each
              rank's stream after a rendezvous, max over ranks), then dra_preempt_batch on one rank
Ranks: --local-world K contexts of this process on ONE device (it measures the protocol, not a speed-up), or one process
per GPU under torchrun.  Prints the card and its power limit, then one JSON line.

  python profiles/shard_preempt.py --local-world 2
  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 profiles/shard_preempt.py
"""
import argparse, importlib, json, os, statistics, subprocess, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §14 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_oracle as P  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
ap = argparse.ArgumentParser()
ap.add_argument("--local-world", type=int, default=0)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
args = ap.parse_args()

dist = None
if args.local_world:
    world, my_ranks, local = args.local_world, list(range(args.local_world)), 0
else:
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    my_ranks = [rank]
dev = torch.device("cuda", local)
lead = my_ranks[0] == 0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(local)


def world_max(x):
    if dist is None:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def world_all(ok):
    if dist is None:
        return ok
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    return int(t.item()) == 0


def dv(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(dev) if a.nbytes else torch.zeros(16, dtype=torch.uint8, device=dev)


def on_streams(ctxs, streams, fn):
    """fn(ctx) on every rank of this process after a device-side rendezvous; the max over ranks of its event time (us)"""
    for c in ctxs:
        c.peer_rendezvous()
    ev = []
    for c, s in zip(ctxs, streams):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s); fn(c); b.record(s); ev.append((a, b))
    for c in ctxs:
        c.sync()
    return world_max(max(a.elapsed_time(b) * 1e3 for a, b in ev))


def median(fn):
    for _ in range(args.warmup):
        fn()
    return statistics.median(fn() for _ in range(args.steps))


def main():
    n_node, n_pod, k = 125, 1000, 16
    rng = np.random.default_rng(1)
    worlds = {
        "cfg2-sized": S.preempt(n_node=n_node, gpus_per_node=8, n_pending=n_pod, seed=1, fill=90, mig_nodes=4, prio_lo=0,
                                prio_hi=1000, pending_prio=1000, shapes=("3g", "7g", "2x3g"),
                                tiles=(R.GI_1_SLICE, R.GI_2_SLICE)),
        "SHARED-heavy": S.preempt(n_node=n_node, gpus_per_node=8, n_pending=n_pod, seed=2, mig_nodes=0, prio_lo=0,
                                  prio_hi=1000, pending_prio=1000, shared_per_gpu=40, shapes=("gpu4",)),
    }
    cands = (rng.integers(0, n_node, n_pod * k).astype(np.uint32), (np.arange(n_pod + 1) * k).astype(np.uint32))
    bounds = [n_node * r // world for r in range(world)] + [n_node]
    if lead:
        print(f"device: {card()}; {world} ranks ({'contexts on one device' if dist is None else 'one GPU each'})")
    streams = [torch.cuda.Stream(device=dev) for _ in my_ranks]
    results, all_ok = [], True
    for wname, w in worlds.items():
        ctxs = [A.Context(device=local, stream=s.cuda_stream) for s in streams]
        for r, c in zip(my_ranks, ctxs):
            if dist is None:
                c.comm_init_local(r, world)
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        if dist is not None:
            uid = [A.Context.comm_unique_id() if lead else None]
            dist.broadcast_object_list(uid, src=0)
            ctxs[0].comm_init(uid[0], my_ranks[0], world)
        for c in ctxs:
            c.set_shard_map(bounds, stray_rank=0)
            c.set_shard_preempt(n_pod, n_pod * n_node, 16)
        if world > 1:
            if dist is None:
                for c in ctxs:
                    c.shard_export(max(1, len(w.run_claims)), 0, want_handle=False)
                for c in ctxs:
                    c.peer_import_local(ctxs)
            else:
                hs = [None] * world
                dist.all_gather_object(hs, ctxs[0].shard_export(max(1, len(w.run_claims))))
                ctxs[0].peer_import(hs)
        keep = [dv(x) for x in (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)]
        run = A.RunningPods(keep[3].data_ptr(), len(w.run_claims), keep[4].data_ptr(), len(w.run_pod_off) - 1,
                            keep[5].data_ptr(), None, keep[6].data_ptr(), len(w.run_out))
        if lead:
            print(f"workload {wname}: {n_node} nodes x 8 GPUs, {len(w.run_pod_off) - 1} running pods, {n_pod} pending pods")
        for form, (cn, co) in (("dense", (None, None)), (f"{k} candidates", cands)):
            n_pair = n_pod * n_node if co is None else int(co[-1])
            d_cn, d_co = (None, None) if cn is None else (dv(cn), dv(co))
            sizes = (n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * 16 * 4)
            outs = [[torch.zeros(s + 16, dtype=torch.uint8, device=dev) for s in sizes] for _ in ctxs]
            for flags in (0, A.F_EXHAUSTIVE):
                what = f"{wname} {form}, flags {'EXHAUSTIVE' if flags else '0'}"
                torch.cuda.synchronize()
                outs_of = {id(c): o for c, o in zip(ctxs, outs)}

                def sharded(c):
                    o = outs_of[id(c)]
                    c.preempt_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                            None if d_cn is None else d_cn.data_ptr(), None if d_co is None else d_co.data_ptr(),
                                            n_pair, run, *[t.data_ptr() for t in o], 16, flags)
                on_streams(ctxs, streams, sharded)
                ref = P.preempt(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                                w.run_prio, w.run_out, None, cn, co, 16, P.F_EXHAUSTIVE if flags else 0)
                dt = (np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32)
                ok = all(all(t.cpu().numpy()[:s].view(d).tobytes() == y.tobytes() for t, s, d, y in zip(o, sizes, dt, ref))
                         for o in outs)
                ok = world_all(ok)
                all_ok = all_ok and ok
                if lead:
                    print(f"oracle check {what}: {'ok' if ok else 'MISMATCH'}")
                if not ok:
                    continue
                t_shard = median(lambda: on_streams(ctxs, streams, sharded))
                single_args = (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co,
                               16, flags)

                def single():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); ctxs[0].preempt(*single_args); b.record(); b.synchronize()
                    return world_max(a.elapsed_time(b) * 1e3)
                t_single = median(single)
                t_sync = median(lambda: on_streams(ctxs, streams, lambda c: c.shard_sync_inventory_device())) if world > 1 else 0.0
                row = dict(workload=wname, form=form, flags=int(flags), pairs=n_pair, sharded_us=round(t_shard, 1),
                           single_us=round(t_single, 1), sync_us=round(t_sync, 1), sync_single_us=round(t_sync + t_single, 1))
                results.append(row)
                if lead:
                    print(f"  {n_pair} pairs: sharded {t_shard / 1e3:8.3f} ms   single {t_single / 1e3:8.3f} ms   "
                          f"sync {t_sync / 1e3:6.3f} + single = {(t_sync + t_single) / 1e3:8.3f} ms")
        torch.cuda.synchronize()
        for c in ctxs:
            c.close()
    if lead:
        print(json.dumps(dict(metric="shard_preempt", world=world, local_world=dist is None, device=card(),
                              oracle_ok=all_ok, cases=results)))
    if dist is not None:
        dist.destroy_process_group()
    sys.exit(0 if all_ok else 1)


if __name__ == "__main__":
    main()
