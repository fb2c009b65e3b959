"""Sharded pod capacity (spec §16 "Sharded form") timings: dra_pod_capacity_batch_global_device at local world 1 and 2,
against the recipe it replaces, the inventory sync on every rank followed by dra_pod_capacity_batch on one rank.  The
workload is profiles/pod_capacity.py's fragmented one: cfg5's fragmented inventory (64 nodes x 8 GPUs) with synth.pods'
20,000 pods of 1..5 MIG claims, dense (1.28 M pairs) and with 16 random candidates per pod (320,000 pairs), first-fit and
DRA_F_EXHAUSTIVE, max_copies 64.  Every case is checked against the CPU oracle on every rank before it is timed.

The world-2 ranks are contexts of this process on ONE device (dra_comm_init_local), so they share its SMs: the figures
show the exchange's overhead, not a multi-GPU speedup.  A figure is the median (min, max) of REPS calls, a host clock
around the enqueue on every rank and the synchronise of every rank.  Prints the card, its power limit and its max SM
clock."""
import importlib
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §16 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import capacity_oracle as K  # noqa: E402

A, S = pkg.api, pkg.synth
REPS = int(os.environ.get("POD_CAPACITY_REPS", "11"))
N_POD = int(os.environ.get("POD_CAPACITY_PODS", "20000"))
MAX_COPIES = 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn):
    fn(); fn()                                                 # warm-up: buffers grown, modules loaded
    ts = []
    for _ in range(REPS):
        t0 = time.perf_counter(); fn(); ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


def dev(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to("cuda:0")


def world_of(w, n, max_pairs):
    """n contexts on device 0, the nodes split evenly"""
    bounds = [w.n_node * r // n for r in range(n)] + [w.n_node]
    ctxs = [A.Context(device=0) for _ in range(n)]
    for r, c in enumerate(ctxs):
        c.comm_init_local(r, n)
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        c.set_shard_map(bounds, stray_rank=0)
        if n > 1:
            c.set_shard_capacity(max_pairs)
            c.shard_export(64, 0, want_handle=False)
    if n > 1:
        for c in ctxs:
            c.peer_import_local(ctxs)
    return ctxs


def main():
    torch.cuda.init()
    print(f"device: {card()}; {REPS} calls per figure")
    w, pod_off = S.pods(n_pod=N_POD)
    rng = np.random.default_rng(1)
    k = 16
    cands = (rng.integers(0, w.n_node, N_POD * k).astype(np.uint32), (np.arange(N_POD + 1) * k).astype(np.uint32))
    d_claims, d_pod_off = dev(w.claims), dev(pod_off)
    worlds = {n: world_of(w, n, N_POD * w.n_node) for n in (1, 2)}
    fails = 0
    for form, (cn, co) in (("dense", (None, None)), (f"{k} candidates", cands)):
        n_pair = N_POD * w.n_node if co is None else int(co[-1])
        d_cn, d_co = (None, None) if cn is None else (dev(cn), dev(co))
        for exhaustive in (False, True):
            flags = A.F_EXHAUSTIVE if exhaustive else 0
            ref = K.capacity(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, MAX_COPIES,
                             K.F_EXHAUSTIVE if exhaustive else 0)
            what = f"fragmented ({w.n_node} nodes x 8 GPUs, {N_POD} pods, {form}), flags {'EXHAUSTIVE' if exhaustive else '0'}"
            print(f"{what}: {n_pair} pairs, {int(ref[2].sum())} copies")
            for n, ctxs in worlds.items():
                outs = [[torch.zeros(s, dtype=torch.uint8, device="cuda:0") for s in (n_pair * 2, n_pair, N_POD * 8, N_POD * 4)]
                        for _ in ctxs]
                torch.cuda.synchronize()

                def call():
                    for c, o in zip(ctxs, outs):
                        c.pod_capacity_global_device(d_claims.data_ptr(), len(w.claims), d_pod_off.data_ptr(), N_POD,
                                                     None if d_cn is None else d_cn.data_ptr(),
                                                     None if d_co is None else d_co.data_ptr(), n_pair, MAX_COPIES,
                                                     *[t.data_ptr() for t in o], flags=flags)
                    for c in ctxs:
                        c.sync()

                call()
                ok = all(t.cpu().numpy().view(r.dtype).tobytes() == r.tobytes() for o in outs for t, r in zip(o, ref))
                fails += not ok
                print(f"  oracle check, sharded call at world {n}: {'ok' if ok else 'MISMATCH'}")
                if ok:
                    t = timed(call)
                    print(f"  sharded call, local world {n}: median {t[0]:9.3f} ms (min {t[1]:.3f}, max {t[2]:.3f})")
            ctxs = worlds[2]
            got = ctxs[0].pod_capacity(w.claims, pod_off, cn, co, MAX_COPIES, exhaustive)
            ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref))
            fails += not ok
            print(f"  oracle check, sync then dra_pod_capacity_batch on rank 0: {'ok' if ok else 'MISMATCH'}")

            def recipe():
                for c in ctxs:
                    c.shard_sync_inventory_device()
                for c in ctxs:
                    c.sync()
                ctxs[0].pod_capacity(w.claims, pod_off, cn, co, MAX_COPIES, exhaustive)

            if ok:
                t = timed(recipe)
                print(f"  inventory sync on both ranks, then dra_pod_capacity_batch (host buffers) on rank 0: "
                      f"median {t[0]:9.3f} ms (min {t[1]:.3f}, max {t[2]:.3f})")
    for ctxs in worlds.values():
        for c in ctxs:
            c.close()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
