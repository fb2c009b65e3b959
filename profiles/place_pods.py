"""Place pods (spec §13) timings on one GPU: dra_place_pods_batch on synth.pods workloads, checked against the CPU oracle
before anything is timed.  Four cases:
  (a) dense candidates (every pod against every node, ascending);
  (b) 8 random candidates per pod;
  (c) the worst case for the visit lists: every pod lists every node in the same order;
  (d) one candidate per pod, the node its claims name, timed next to dra_allocate_pods_batch on the same input.
Each time is the median of repeated calls, CUDA events around the call (host buffers in, host buffers out, as a caller
sees it), every call from the same starting inventory (DRA_F_FRESH_INVENTORY).  Prints the card and its power limit."""
import importlib
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §13 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import place_oracle as P  # noqa: E402

A, S = pkg.api, pkg.synth
REPS = int(os.environ.get("PLACE_REPS", "20"))


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
    flags = A.F_EXHAUSTIVE | A.F_FRESH_INVENTORY
    n_pod, n_node = 20_000, 64
    w, pod_off = S.pods(n_pod, n_node, 1)
    n_pod = len(pod_off) - 1
    rng = np.random.default_rng(1)
    cases = {
        "(a) dense": (None, None),
        "(b) 8 random candidates": (rng.integers(0, n_node, n_pod * 8).astype(np.uint32),
                                    (np.arange(n_pod + 1) * 8).astype(np.uint32)),
        "(c) every node, same order": (np.tile(np.arange(n_node, dtype=np.uint32), n_pod),
                                       (np.arange(n_pod + 1) * n_node).astype(np.uint32)),
        "(d) one candidate (own node)": (w.claims["node"][pod_off[:-1]].astype(np.uint32),
                                         np.arange(n_pod + 1, dtype=np.uint32)),
    }
    print(f"workload: synth.pods({n_pod} pods, {len(w.claims)} claims, {n_node} nodes x 8 GPUs), DRA_F_EXHAUSTIVE, "
          f"{REPS} calls per case")
    with A.Context(device=0) as ctx:
        ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
        for name, (cn, co) in cases.items():                 # correctness first
            out, pod_node = ctx.place_pods(w.claims, pod_off, cn, co, flags=flags)
            ref, ref_node, inv = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, flags=P.F_EXHAUSTIVE)
            ok = out.tobytes() == ref.tobytes() and pod_node.tobytes() == ref_node.tobytes() and \
                ctx.get_inventory().tobytes() == inv.tobytes()
            print(f"oracle check {name:<30} {'ok' if ok else 'MISMATCH'}: {int((pod_node != 0xFFFFFFFF).sum())}/{n_pod} pods placed")
            if not ok:
                sys.exit(1)
        ref_pods = ctx.allocate_pods(w.claims, pod_off, flags=flags)
        if ref_pods.tobytes() != ctx.place_pods(w.claims, pod_off, *cases["(d) one candidate (own node)"], flags=flags)[0].tobytes():
            print("(d) differs from dra_allocate_pods_batch"); sys.exit(1)
        for name, (cn, co) in cases.items():
            med, lo, hi = timed(lambda: ctx.place_pods(w.claims, pod_off, cn, co, flags=flags))
            print(f"{name:<32} place_pods      median {med:9.1f} us  (min {lo:.1f}, max {hi:.1f})")
        med, lo, hi = timed(lambda: ctx.allocate_pods(w.claims, pod_off, flags=flags))
        print(f"{'(d) same input':<32} allocate_pods   median {med:9.1f} us  (min {lo:.1f}, max {hi:.1f})")


if __name__ == "__main__":
    main()
