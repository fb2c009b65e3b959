"""Why each node is unsuitable (spec §17) against UnsuitableNodes (§8) on one GPU: dra_unsuitable_why_batch and
dra_unsuitable_batch through host buffers on the same pairs with the same flags.  Workloads:
  cfg2 half-full  bench_unsuitable.py's: cfg2's inventory after its first 4,000 claims, 10,000 one-claim pods, dense
                  (1.25 M pairs);
  fragmented      cfg5's fragmented inventory (64 nodes x 8 GPUs) with synth.pods' 20,000 pods of 1..5 MIG claims, dense
                  (1.28 M pairs).
Each with flags 0 and DRA_F_EXHAUSTIVE; the reasons call with the tallies (pod_why, claim_blocks) and without them (the
pair records only).  Before timing, each case checks that the reason is OK exactly where the bit is set.  A call's time
is the median (min, max) of REPS calls, CUDA events around the synchronising host-buffer call, outputs read back
included.  Prints the card, its power limit and its max SM clock."""
import importlib
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("k8s-dra-driver_b200")
from oracle import oracle as O  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("UNSUITABLE_WHY_REPS", "11"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn):
    fn(); fn()                                                 # warm-up: buffers grown, modules loaded
    ts = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts), max(ts)


def case(ctx, name, claims, pod_off):
    for exh in (False, True):
        flags = A.F_EXHAUSTIVE if exh else 0
        bits = ctx.unsuitable(claims, pod_off, None, None, flags)
        why = ctx.unsuitable_why(claims, pod_off, exhaustive=exh)[0]
        ok = np.unpackbits(np.asarray(bits, np.uint8), bitorder="little")[:len(why)].astype(bool)
        if not (ok == (why == R.ST_OK)).all():
            print(f"{name}: reasons disagree with the bits"); sys.exit(1)
        counts = np.bincount(why, minlength=A.WHY_N)
        uns = timed(lambda: ctx.unsuitable(claims, pod_off, None, None, flags))
        full = timed(lambda: ctx.unsuitable_why(claims, pod_off, exhaustive=exh))
        bare = timed(lambda: ctx.unsuitable_why(claims, pod_off, exhaustive=exh, want_claims=False, want_tallies=False))
        print(f"{name}, flags {'EXHAUSTIVE' if exh else '0'}: {len(why)} pairs, reasons {counts.tolist()}")
        print(f"  unsuitable (bits)            median {uns[0]:8.3f} ms (min {uns[1]:.3f}, max {uns[2]:.3f})")
        print(f"  unsuitable_why, all outputs  median {full[0]:8.3f} ms (min {full[1]:.3f}, max {full[2]:.3f})")
        print(f"  unsuitable_why, reasons only median {bare[0]:8.3f} ms (min {bare[1]:.3f}, max {bare[2]:.3f})")


def main():
    torch.cuda.init()
    print(f"device: {card()}; {REPS} calls per figure")
    with A.Context(device=0) as ctx:
        w = S.cfg2()
        _, inv = O.allocate(w.gpus, w.node_off, w.table, w.claims[:4000])
        ctx.set_table(w.table); ctx.set_inventory(inv, w.node_off)
        n_pod = 10_000
        case(ctx, f"cfg2 half-full ({w.n_node} nodes, {n_pod} pods, dense)", w.claims[:n_pod].copy(),
             np.arange(n_pod + 1, dtype=np.uint32))
        w, pod_off = S.pods(n_pod=20_000)
        ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
        case(ctx, f"fragmented ({w.n_node} nodes, {len(pod_off) - 1} pods of 1..5 MIG claims, dense)", w.claims, pod_off)


if __name__ == "__main__":
    main()
