"""Sharded reasons of UnsuitableNodes (spec §17 "Sharded form") timings: dra_unsuitable_why_batch_global_device at local
world 1 and 2, against the recipe it replaces (the inventory sync on every rank, then dra_unsuitable_why_batch on one
rank) and against the sharded bits call (dra_unsuitable_batch_global_device) on the same pairs.  The workload is the
fragmented one of profiles/unsuitable_why.py: cfg5's fragmented inventory (64 nodes x 8 GPUs) with synth.pods' 20,000 pods
of 1..5 MIG claims, dense (1.28 M pairs) and with 16 random candidates per pod (320,000 pairs), first-fit and
DRA_F_EXHAUSTIVE, all four outputs.

Before a case is timed, every rank's four outputs are checked byte for byte against dra_unsuitable_why_batch on a rank
holding the world after the inventory sync, and the pairs of SAMPLE pods spread over the batch against the CPU oracle
(tests/why_oracle.py; the whole batch would take the exhaustive oracle most of an hour).

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
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §17 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import why_oracle as Y  # noqa: E402

A, S = pkg.api, pkg.synth
REPS = int(os.environ.get("UNSUITABLE_WHY_REPS", "11"))
N_POD = int(os.environ.get("UNSUITABLE_WHY_PODS", "20000"))
SAMPLE = int(os.environ.get("UNSUITABLE_WHY_SAMPLE", "32"))


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
    """n contexts on device 0, the nodes split evenly, with room for the reasons and the bits calls"""
    bounds = [w.n_node * r // n for r in range(n)] + [w.n_node]
    ctxs = [A.Context(device=0) for _ in range(n)]
    for r, c in enumerate(ctxs):
        c.comm_init_local(r, n)
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        c.set_shard_map(bounds, stray_rank=0)
        if n > 1:
            c.set_shard_why(max_pairs)
            c.set_shard_pairs(max_pairs)
            c.shard_export(64, 0, want_handle=False)
    if n > 1:
        for c in ctxs:
            c.peer_import_local(ctxs)
    return ctxs


def sampled(w, pod_off, cn, co, exhaustive, got):
    """The pairs of SAMPLE pods spread over the batch against the CPU oracle: True when all agree."""
    for p in np.linspace(0, N_POD - 1, SAMPLE).astype(np.int64):
        k0, k1 = (p * w.n_node, (p + 1) * w.n_node) if co is None else (int(co[p]), int(co[p + 1]))
        one = np.array([pod_off[p], pod_off[p + 1]], np.uint32)
        nodes = np.arange(w.n_node, dtype=np.uint32) if co is None else cn[k0:k1]
        ref = Y.why(w.gpus, w.node_off, w.table, w.claims, one, nodes, np.array([0, len(nodes)], np.uint32),
                    Y.F_EXHAUSTIVE if exhaustive else 0)
        if got[0][k0:k1].tobytes() != ref[0].tobytes() or got[1][k0:k1].tobytes() != ref[1].tobytes() or \
                got[2][p].tobytes() != ref[2][0].tobytes():
            return False
    return True


def main():
    torch.cuda.init()
    print(f"device: {card()}; {REPS} calls per figure")
    w, pod_off = S.pods(n_pod=N_POD)
    rng = np.random.default_rng(1)
    k = 16
    cands = (rng.integers(0, w.n_node, N_POD * k).astype(np.uint32), (np.arange(N_POD + 1) * k).astype(np.uint32))
    d_claims, d_pod_off = dev(w.claims), dev(pod_off)
    n_claim = len(w.claims)
    worlds = {n: world_of(w, n, N_POD * w.n_node) for n in (1, 2)}
    fails = 0
    for form, (cn, co) in (("dense", (None, None)), (f"{k} candidates", cands)):
        n_pair = N_POD * w.n_node if co is None else int(co[-1])
        d_cn, d_co = (None, None) if cn is None else (dev(cn), dev(co))
        for exhaustive in (False, True):
            flags = A.F_EXHAUSTIVE if exhaustive else 0
            ctxs = worlds[2]
            for c in ctxs:
                c.shard_sync_inventory_device()
            for c in ctxs:
                c.sync()
            ref = ctxs[0].unsuitable_why(w.claims, pod_off, cn, co, exhaustive)
            ok = sampled(w, pod_off, cn, co, exhaustive, ref)
            fails += not ok
            what = f"fragmented ({w.n_node} nodes x 8 GPUs, {N_POD} pods, {form}), flags {'EXHAUSTIVE' if exhaustive else '0'}"
            print(f"{what}: {n_pair} pairs, reasons {np.bincount(ref[0], minlength=A.WHY_N).tolist()}")
            print(f"  oracle check of {SAMPLE} pods, sync then dra_unsuitable_why_batch on rank 0: {'ok' if ok else 'MISMATCH'}")
            sizes = (n_pair, n_pair * 4, N_POD * A.WHY_N * 4, n_claim * 4)
            for n, ctxs in worlds.items():
                outs = [[torch.zeros(s, dtype=torch.uint8, device="cuda:0") for s in sizes] for _ in ctxs]
                bits = [torch.zeros((n_pair + 7) // 8, dtype=torch.uint8, device="cuda:0") for _ in ctxs]
                torch.cuda.synchronize()

                def call():
                    for c, o in zip(ctxs, outs):
                        c.unsuitable_why_global_device(d_claims.data_ptr(), n_claim, d_pod_off.data_ptr(), N_POD,
                                                       None if d_cn is None else d_cn.data_ptr(),
                                                       None if d_co is None else d_co.data_ptr(), n_pair,
                                                       *[t.data_ptr() for t in o], flags=flags)
                    for c in ctxs:
                        c.sync()

                def call_bits():
                    for c, b in zip(ctxs, bits):
                        c.unsuitable_global_device(d_claims.data_ptr(), n_claim, d_pod_off.data_ptr(), N_POD,
                                                   None if d_cn is None else d_cn.data_ptr(),
                                                   None if d_co is None else d_co.data_ptr(), n_pair, b.data_ptr(), flags)
                    for c in ctxs:
                        c.sync()

                call()
                call_bits()
                ok = all(t.cpu().numpy().tobytes() == np.ascontiguousarray(r).view(np.uint8).tobytes()
                         for o in outs for t, r in zip(o, ref))
                ok_bits = all(np.unpackbits(b.cpu().numpy(), bitorder="little")[:n_pair].astype(bool).tobytes() ==
                              (ref[0] == Y.ST_OK).tobytes() for b in bits)
                fails += not (ok and ok_bits)
                print(f"  check, sharded call at world {n} against the synced single call: {'ok' if ok else 'MISMATCH'}; "
                      f"OK against the sharded bits: {'ok' if ok_bits else 'MISMATCH'}")
                if ok and ok_bits:
                    t = timed(call)
                    print(f"  sharded reasons, local world {n}: median {t[0]:9.3f} ms (min {t[1]:.3f}, max {t[2]:.3f})")
                    t = timed(call_bits)
                    print(f"  sharded bits,    local world {n}: median {t[0]:9.3f} ms (min {t[1]:.3f}, max {t[2]:.3f})")
            ctxs = worlds[2]

            def recipe():
                for c in ctxs:
                    c.shard_sync_inventory_device()
                for c in ctxs:
                    c.sync()
                ctxs[0].unsuitable_why(w.claims, pod_off, cn, co, exhaustive)

            t = timed(recipe)
            print(f"  inventory sync on both ranks, then dra_unsuitable_why_batch (host buffers) on rank 0: "
                  f"median {t[0]:9.3f} ms (min {t[1]:.3f}, max {t[2]:.3f})")
    for ctxs in worlds.values():
        for c in ctxs:
            c.close()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
