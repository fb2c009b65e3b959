"""Preemption (spec §14) timings on one GPU: dra_preempt_batch on synth.preempt worlds, every case checked against the CPU
oracle before anything is timed.  Workloads:
  cfg2-sized    125 nodes x 8 MIG GPUs, ~90 % taken by 1g and 2g running pods at priorities 0..999, 1,000 pending 3g, 7g
                and 2x3g pods at priority 1000; dense (125,000 pairs) and 16 random candidates per pod, each with and
                without DRA_F_EXHAUSTIVE;
  SHARED-heavy  125 non-MIG nodes x 8 GPUs carrying up to 40 time-slicing / MPS pods each, 1,000 pending 4-GPU pods.
Each time is the median (min, max) of repeated calls, CUDA events around the host-buffer call, next to the CPU oracle's
single-thread time on the same input (one call).  Prints the card and its power limit."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §14 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_oracle as P  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("PREEMPT_REPS", "10"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn):
    fn()                                                       # warm-up: buffers grown, modules loaded
    ts = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


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
            print(f"workload {wname}: {n_node} nodes x 8 GPUs, {len(w.run_pod_off) - 1} running pods, {n_pod} pending pods")
            ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
            for form, (cn, co) in (("dense", (None, None)), (f"{k} candidates", cands)):
                for flags in (0, A.F_EXHAUSTIVE):
                    args = (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co, 16, flags)
                    got = ctx.preempt(*args)
                    t0 = time.perf_counter()
                    ref = P.preempt(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                                    w.run_prio, w.run_out, None, cn, co, 16, P.F_EXHAUSTIVE if flags else 0)
                    t_cpu = time.perf_counter() - t0
                    ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and \
                        ctx.get_inventory().tobytes() == w.gpus.tobytes()
                    n_pair = len(got[0])
                    what = f"{wname} {form}, flags {'EXHAUSTIVE' if flags else '0'}"
                    print(f"oracle check {what}: {'ok' if ok else 'MISMATCH'} (pods FITS {int((got[3] == 0).sum())}, "
                          f"EVICT {int((got[3] == 1).sum())}, other {int((got[3] > 1).sum())})")
                    if not ok:
                        sys.exit(1)
                    med, lo, hi = timed(lambda: ctx.preempt(*args))
                    print(f"  {n_pair} pairs: median {med / 1e3:9.2f} ms (min {lo / 1e3:.2f}, max {hi / 1e3:.2f}), "
                          f"{n_pair / (med * 1e-6):.3g} pairs/s; CPU oracle, one thread: {t_cpu * 1e3:.0f} ms")


if __name__ == "__main__":
    main()
