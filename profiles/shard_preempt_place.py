"""Sharded preempt and place (spec §15, "Sharded form") on one GPU shared by K world contexts, every case checked against
the CPU oracle before anything is timed.  Workload: the cfg2-sized preemption world of profiles/preempt_place.py (125 nodes
x 8 MIG GPUs, ~90 % taken by running pods at priorities 0..999, 1,000 pending pods at priority 1000), dense and with 16
random candidates per pod, first-fit.  Each rank starts from the real world on its own range and empty nodes elsewhere.
Reported, median (min, max) of repeated calls on the host clock from the first enqueue to the last rank's sync, every
inventory reloaded (untimed) before each:
  sharded     dra_preempt_place_batch_global_device on every rank
  single      dra_preempt_place_batch on one context holding the whole world (host buffers)
  workaround  what a sharded world needed without the call: dra_shard_sync_inventory_device on every rank, then
              dra_preempt_place_batch on rank 0, dra_get_inventory of its result and dra_set_inventory on every rank
With K contexts on one GPU they share its SMs: this measures the protocol's cost, not a speed-up.
  python profiles/shard_preempt_place.py --local-world 1 2 4
Prints the card, its power limit and its max SM clock."""
import argparse
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
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §15 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_place_oracle as PP  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("SHARD_PREEMPT_PLACE_REPS", "7"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def dv(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to("cuda:0") if a.nbytes else torch.zeros(16, dtype=torch.uint8, device="cuda:0")


def stats(ts):
    return f"{statistics.median(ts):9.1f} us ({min(ts):.1f} .. {max(ts):.1f})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--local-world", type=int, nargs="+", default=[1, 2, 4])
    args = ap.parse_args()
    print(card())
    w = S.preempt(n_node=125, gpus_per_node=8, n_pending=1000, seed=12, mig_nodes=4)
    n_node, n_pod, n_run = 125, len(w.pod_off) - 1, len(w.run_pod_off) - 1
    placed = w.claims.copy(); placed["node"] = 0
    sl = R.claim_slots(placed, 1).astype(np.int64)
    oo = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32)
    n_out = int(sl.sum())
    rng = np.random.default_rng(12)
    forms = {"dense": (None, None),
             "16 random": (rng.integers(0, n_node, n_pod * 16).astype(np.uint32), (np.arange(n_pod + 1) * 16).astype(np.uint32))}
    keep = [dv(x) for x in (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, oo)]
    run = A.RunningPods(keep[3].data_ptr(), len(w.run_claims), keep[4].data_ptr(), n_run, keep[5].data_ptr(), None,
                        keep[6].data_ptr(), len(w.run_out))
    for name, (cn, co) in forms.items():
        ref = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                               w.run_prio, w.run_out, None, cn, co, oo, n_out, 0)
        print(f"\n{name}: {n_pod} pods, {int((ref[2] == PP.EVICT).sum())} evicting, {int((ref[1] != 0xFFFFFFFF).sum())} placed")
        with A.Context(device=0) as single:
            single.set_table(w.table)
            def one():
                return single.preempt_place(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                                            None, cn, co, oo, n_out, 0)
            single.set_inventory(w.gpus, w.node_off)
            got = one()
            assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref[:4])), "single call differs from the oracle"
            ts = []
            for _ in range(REPS):
                single.set_inventory(w.gpus, w.node_off)
                t0 = time.perf_counter(); one(); ts.append((time.perf_counter() - t0) * 1e6)
            print(f"  single      K=1  {stats(ts)}")
        d_n, d_o = (dv(cn), dv(co)) if cn is not None else (None, None)
        for K in args.local_world:
            bounds = [n_node * r // K for r in range(K)] + [n_node]
            invs = []
            for r in range(K):
                g = w.empty.copy()
                a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
                g[a:b] = w.gpus[a:b]
                invs.append(g)
            ctxs = [A.Context(device=0) for _ in range(K)]
            try:
                for r, c in enumerate(ctxs):
                    c.comm_init_local(r, K); c.set_table(w.table); c.set_inventory(invs[r], w.node_off)
                    c.set_shard_map(bounds, 0)
                    if K > 1:
                        c.set_shard_preempt_place(n_pod, n_pod * n_node, n_run)
                        c.shard_export(n_out, 0, want_handle=False)
                if K > 1:
                    for c in ctxs:
                        c.peer_import_local(ctxs)
                outs = [[torch.zeros(s, dtype=torch.uint8, device="cuda:0") for s in (n_pod * 4, n_pod, n_run * 4)] for _ in ctxs]
                torch.cuda.synchronize()

                def reload():
                    for r, c in enumerate(ctxs):
                        c.set_inventory(invs[r], w.node_off)

                def sharded():
                    for c, o in zip(ctxs, outs):
                        c.preempt_place_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(),
                                                      n_pod, d_n.data_ptr() if d_n is not None else None,
                                                      d_o.data_ptr() if d_o is not None else None, 0 if co is None else int(co[-1]),
                                                      run, keep[7].data_ptr(), n_out, *[t.data_ptr() for t in o], 0)
                    for c in ctxs:
                        c.sync()

                reload(); sharded()
                for r, (c, o) in enumerate(zip(ctxs, outs)):
                    table = c.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE))
                    got = [table] + [t.cpu().numpy().view(d) for t, d in zip(o, (np.uint32, np.uint8, np.uint32))]
                    assert all(x.tobytes() == y.tobytes() for x, y in zip(got, ref[:4])), f"K={K} rank {r} differs from the oracle"
                    a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
                    assert c.get_inventory()[a:b].tobytes() == ref[4][a:b].tobytes(), f"K={K} rank {r} inventory"
                ts = []
                for _ in range(REPS):
                    reload()
                    t0 = time.perf_counter(); sharded(); ts.append((time.perf_counter() - t0) * 1e6)
                print(f"  sharded     K={K}  {stats(ts)}")
                if K > 1:
                    def workaround():
                        for c in ctxs:
                            c.shard_sync_inventory_device()
                        for c in ctxs:
                            c.sync()
                        ctxs[0].preempt_place(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio,
                                              w.run_out, None, cn, co, oo, n_out, 0)
                        g = ctxs[0].get_inventory()
                        for c in ctxs:
                            c.set_inventory(g, w.node_off)
                    reload(); workaround()
                    assert ctxs[K - 1].get_inventory().tobytes() == ref[4].tobytes(), "workaround differs from the oracle"
                    ts = []
                    for _ in range(REPS):
                        reload()
                        t0 = time.perf_counter(); workaround(); ts.append((time.perf_counter() - t0) * 1e6)
                    print(f"  workaround  K={K}  {stats(ts)}")
            finally:
                for c in ctxs:
                    c.close()


if __name__ == "__main__":
    main()
