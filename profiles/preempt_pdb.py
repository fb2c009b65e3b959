"""Preemption with disruption budgets (spec §14, "Disruption budgets") against preemption without them, on one GPU: the
worlds of profiles/preempt.py (cfg2-sized MIG, SHARED-heavy), dense and 16 random candidates, flags 0.  Per case three
calls on the same seeded problem, timed alternately in one loop:
  dra_preempt_batch                     the budget-free call
  dra_preempt_pdb_batch, no budgets     NULL budgets: must cost what the budget-free call costs
  dra_preempt_pdb_batch, budgets        8 budgets over the running pods (1 in 4 pods in none), allowed 0..3
Each output is first checked byte for byte against the CPU oracle (tests/pod_oracles.c).  Times are medians (min, max)
of CUDA events around the host-buffer call.  Prints the card and its power limit."""
import importlib
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §14 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_oracle as P  # noqa: E402
import preempt_oracle as PB  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("PREEMPT_REPS", "10"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def event_us(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); b.synchronize()
    return a.elapsed_time(b) * 1e3


def main():
    torch.cuda.init()
    print(f"device: {card()}")
    n_node, n_pod = 125, 1000
    rng = np.random.default_rng(1)
    worlds = {
        "cfg2-sized": S.preempt(n_node=n_node, gpus_per_node=8, n_pending=n_pod, seed=1, fill=90, mig_nodes=4, prio_lo=0,
                                prio_hi=1000, pending_prio=1000, shapes=("3g", "7g", "2x3g"),
                                tiles=(R.GI_1_SLICE, R.GI_2_SLICE)),
        "SHARED-heavy": S.preempt(n_node=n_node, gpus_per_node=8, n_pending=n_pod, seed=2, mig_nodes=0, prio_lo=0,
                                  prio_hi=1000, pending_prio=1000, shared_per_gpu=40, shapes=("gpu4",)),
    }
    k = 16
    cands = (rng.integers(0, n_node, n_pod * k).astype(np.uint32), (np.arange(n_pod + 1) * k).astype(np.uint32))
    with A.Context(device=0) as ctx:
        for wname, w in worlds.items():
            n_run = len(w.run_pod_off) - 1
            run_pdb = rng.integers(0, 8, n_run).astype(np.uint32)
            run_pdb[rng.integers(0, 4, n_run) == 0] = A.PDB_NONE
            allowed = rng.integers(0, 4, 8).astype(np.int32)
            print(f"workload {wname}: {n_node} nodes x 8 GPUs, {n_run} running pods, {n_pod} pending pods, 8 budgets")
            ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
            for form, (cn, co) in (("dense", (None, None)), (f"{k} candidates", cands)):
                run = (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
                calls = {
                    "dra_preempt_batch": lambda: ctx.preempt(*run, None, cn, co, 16, 0),
                    "dra_preempt_pdb_batch, no budgets": lambda: ctx.preempt_pdb(*run, None, None, None, cn, co, 16, 0),
                    "dra_preempt_pdb_batch, budgets": lambda: ctx.preempt_pdb(*run, run_pdb, allowed, None, cn, co, 16, 0),
                }
                oracle = (PB.preempt_pdb(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                                        w.run_pod_off, w.run_prio, w.run_out, None, None, None, cn, co, 16, 0),
                          PB.preempt_pdb(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                                        w.run_pod_off, w.run_prio, w.run_out, run_pdb, allowed, None, cn, co, 16, 0))
                for i, (name, fn) in enumerate(calls.items()):
                    ref = oracle[0][:6] if i == 0 else oracle[i - 1]
                    ok = all(x.tobytes() == y.tobytes() for x, y in zip(fn(), ref))
                    print(f"oracle check {wname} {form}, {name}: {'ok' if ok else 'MISMATCH'}")
                    if not ok:
                        sys.exit(1)
                got = oracle[1]
                print(f"  with budgets: EVICT pods {int((got[3] == 1).sum())}, violating victims of the chosen pairs "
                      f"{int(got[7].sum())}, EVICT pairs with a violation {int((got[6] > 0).sum())}")
                ts = {name: [] for name in calls}
                for _ in range(REPS):                      # alternated, so the three see the same machine
                    for name, fn in calls.items():
                        ts[name].append(event_us(fn))
                for name, t in ts.items():
                    print(f"  {form:14s} {name:36s} median {statistics.median(t) / 1e3:8.2f} ms "
                          f"(min {min(t) / 1e3:.2f}, max {max(t) / 1e3:.2f})")


if __name__ == "__main__":
    main()
