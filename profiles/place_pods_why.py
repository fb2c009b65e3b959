"""Why place pods put each pod where it did (spec §18): dra_place_pods_why_batch timed against dra_place_pods_batch on
profiles/place_pods.py's workloads (a)-(d), alternating the two calls in one run.  Before anything is timed, each case
is checked: out, pod_node and the inventory against the CPU oracle of §13, every pod's node against its first OK pair,
and the pairs of sampled pods against the §18 oracle on the inventory the pods before them left.  Each time is the median
of repeated calls, CUDA events around the call (host buffers in, host buffers out), every call from the same starting
inventory (DRA_F_FRESH_INVENTORY).  Prints the card, its power limit and SM clock."""
import importlib
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracles of spec §13 / §18 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import place_oracle as P  # noqa: E402
import place_why_oracle as PW  # noqa: E402
import why_oracle as Y  # noqa: E402

A, S = pkg.api, pkg.synth
REPS = int(os.environ.get("PLACE_REPS", "20"))
NONE = 0xFFFFFFFF


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def check(ctx, w, pod_off, cn, co, flags, name):
    out, pod_node, why, claim, _, _ = ctx.place_pods_why(w.claims, pod_off, cn, co, flags=flags)
    ref, ref_node, inv = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, flags=P.F_EXHAUSTIVE)
    ok = out.tobytes() == ref.tobytes() and pod_node.tobytes() == ref_node.tobytes() and \
        ctx.get_inventory().tobytes() == inv.tobytes()
    n_pod, n_node = len(pod_off) - 1, w.n_node
    k0 = (np.arange(n_pod + 1) * n_node).astype(np.int64) if co is None else co.astype(np.int64)
    nodes = np.tile(np.arange(n_node, dtype=np.uint32), n_pod) if co is None else cn
    for p in range(n_pod):                                     # consequence 1
        hit = np.flatnonzero(why[k0[p]:k0[p + 1]] == Y.ST_OK)
        cnt = int(pod_off[p + 1] - pod_off[p])
        if 0 < cnt <= Y.MAX_POD:
            ok = ok and int(pod_node[p]) == (int(nodes[k0[p] + hit[0]]) if len(hit) else NONE)
    for p in np.random.default_rng(7).choice(n_pod, 4, replace=False).tolist() + [n_pod - 1]:   # sampled pods on W_p
        c0 = int(pod_off[p])
        _, _, live = P.place_pods(w.gpus, w.node_off, w.table, w.claims[:c0], pod_off[:p + 1], cn,
                                  None if co is None else co[:p + 1], flags=P.F_EXHAUSTIVE)
        for k in range(k0[p], k0[p + 1]):
            r, c = PW.pair_reason(live, w.node_off, w.table, w.claims, c0, int(pod_off[p + 1]), int(nodes[k]), None,
                                  None, True, False)
            ok = ok and (int(why[k]), int(claim[k])) == (r, c)
    print(f"oracle check {name:<30} {'ok' if ok else 'MISMATCH'}: {int((pod_node != NONE).sum())}/{n_pod} pods placed, "
          f"{len(why)} pairs")
    if not ok:
        sys.exit(1)


def main():
    torch.cuda.init()
    print(f"device (name, power limit, SM clock, max SM clock): {card()}")
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
          f"{REPS} calls per case and call, alternating")
    with A.Context(device=0) as ctx:
        ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
        for name, (cn, co) in cases.items():                 # correctness first
            check(ctx, w, pod_off, cn, co, flags, name)
        for name, (cn, co) in cases.items():
            calls = {"place_pods": lambda: ctx.place_pods(w.claims, pod_off, cn, co, flags=flags),
                     "place_pods_why": lambda: ctx.place_pods_why(w.claims, pod_off, cn, co, flags=flags),
                     "place_pods_why (reasons only)": lambda: ctx.place_pods_why(w.claims, pod_off, cn, co, flags=flags,
                                                                                 want_claims=False, want_tallies=False)}
            for fn in calls.values():
                fn()                                           # warm-up: buffers grown, modules loaded
            ts = {k: [] for k in calls}
            for _ in range(REPS):
                for k, fn in calls.items():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(); fn(); b.record(); b.synchronize()
                    ts[k].append(a.elapsed_time(b) * 1e3)
            base = statistics.median(ts["place_pods"])
            for k, v in ts.items():
                med = statistics.median(v)
                print(f"{name:<30} {k:<30} median {med:9.1f} us  (min {min(v):.1f}, max {max(v):.1f})  x{med / base:.2f}")
    print(f"device after the run: {card()}")


if __name__ == "__main__":
    main()
