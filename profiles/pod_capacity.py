"""Pod capacity (spec §16) timings on one GPU: dra_pod_capacity_batch through host buffers, every case checked against the
CPU oracle before anything is timed.  Workloads:
  instances free  cfg2's inventory (125 nodes x 8 empty MIG GPUs), dense, six one-claim pods (1g, 2g, 3g, 7g, a whole GPU,
                  a time-slicing share): the per-node "instances free" table, 750 pairs, max_copies 64;
  fragmented      cfg5's fragmented inventory (64 nodes x 8 GPUs) with synth.pods' 20,000 pods of 1..5 MIG claims, dense
                  (1.28 M pairs) and with 16 random candidates per pod (320,000 pairs), first-fit and DRA_F_EXHAUSTIVE,
                  max_copies 64.
Beside each: dra_unsuitable_batch on the same pairs with the same flags (one evaluation per pair) and the CPU oracle on
one thread.  A call's time is the median (min, max) of REPS calls, CUDA events around the synchronising host-buffer call.
Prints the card, its power limit and its max SM clock."""
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

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("POD_CAPACITY_REPS", "11"))
N_POD = int(os.environ.get("POD_CAPACITY_PODS", "20000"))


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


def case(ctx, name, w, claims, pod_off, cn, co, exhaustive, max_copies=64):
    got = ctx.pod_capacity(claims, pod_off, cn, co, max_copies, exhaustive)
    t0 = time.perf_counter()
    ref = K.capacity(w.gpus, w.node_off, w.table, claims, pod_off, cn, co, max_copies, K.F_EXHAUSTIVE if exhaustive else 0)
    t_cpu = time.perf_counter() - t0
    ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and ctx.get_inventory().tobytes() == w.gpus.tobytes()
    what = f"{name}, flags {'EXHAUSTIVE' if exhaustive else '0'}"
    print(f"oracle check {what}: {'ok' if ok else 'MISMATCH'} ({len(got[0])} pairs, {int(got[0].astype(np.int64).sum())} "
          f"copies, {int((got[0] > 0).sum())} pairs with a copy, {int((got[1] == R.ST_SEARCH_LIMIT).sum())} SEARCH_LIMIT)")
    if not ok:
        sys.exit(1)
    flags = A.F_EXHAUSTIVE if exhaustive else 0
    cap = timed(lambda: ctx.pod_capacity(claims, pod_off, cn, co, max_copies, exhaustive))
    uns = timed(lambda: ctx.unsuitable(claims, pod_off, cn, co, flags))
    print(f"  pod_capacity: median {cap[0]:9.3f} ms (min {cap[1]:.3f}, max {cap[2]:.3f}); unsuitable on the same pairs: "
          f"median {uns[0]:9.3f} ms (min {uns[1]:.3f}, max {uns[2]:.3f}); CPU oracle, one thread: {t_cpu * 1e3:.0f} ms")


def main():
    torch.cuda.init()
    print(f"device: {card()}; {REPS} calls per figure")
    with A.Context(device=0) as ctx:
        w = S.cfg2()
        c = np.zeros(6, R.CLAIM_DTYPE)
        c["kind"], c["count"] = R.KIND_MIG, 1
        c["profile"][:4] = [R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_7_SLICE]
        c["kind"][4:] = [R.KIND_GPU, R.KIND_SHARED]
        ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
        case(ctx, f"instances free ({w.n_node} nodes x 8 GPUs, 6 pods, dense)", w, c, np.arange(7, dtype=np.uint32), None, None, False)

        w, pod_off = S.pods(n_pod=N_POD)
        rng = np.random.default_rng(1)
        k = 16
        cands = (rng.integers(0, w.n_node, N_POD * k).astype(np.uint32), (np.arange(N_POD + 1) * k).astype(np.uint32))
        ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
        for form, (cn, co) in (("dense", (None, None)), (f"{k} candidates", cands)):
            for exhaustive in (False, True):
                case(ctx, f"fragmented ({w.n_node} nodes x 8 GPUs, {N_POD} pods, {form})", w, w.claims, pod_off, cn, co, exhaustive)


if __name__ == "__main__":
    main()
