"""Why preemption judged each node as it did (spec §19): dra_preempt_why_batch timed against dra_preempt_batch, and
dra_preempt_place_why_batch against dra_preempt_place_batch, on the worlds of profiles/preempt.py and
profiles/preempt_place.py (cfg2-sized and SHARED-heavy: 125 nodes x 8 GPUs, 1,000 pending pods), dense and 16 random
candidates per pod, each with and without DRA_F_EXHAUSTIVE.  Before anything is timed, each case is checked: the statuses
against the plain call's (dra_preempt_batch's pair_status; dra_preempt_place_batch's out, pod_node, pod_status,
evicted_by and inventory), and the pairs of sampled pods against the §19 oracle (for §15 on the inventory and running pods
the pods before them left).  Each time is the median (min, max) of repeated calls, CUDA events around the host-buffer
call, the two calls of a pair alternated, the live inventory reset before each §15 call.  The §14 reasons call runs no
reprieve, no choice and no victim rows.  Prints the card, its power limit and its max SM clock."""
import importlib
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracles of spec §14 / §15 / §19 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_place_oracle as PP  # noqa: E402
import preempt_why_oracle as PY  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("PREEMPT_WHY_REPS", "7"))
NONE = 0xFFFFFFFF


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def one_pod(w, p, gpus, alive, cands):
    """the §19 oracle's §14 form for pod p alone, on gpus with the running pods `alive`"""
    c0, c1 = int(w.pod_off[p]), int(w.pod_off[p + 1])
    keep = np.isin(np.repeat(np.arange(len(w.run_pod_off) - 1), np.diff(w.run_pod_off)), alive)
    rpo = np.concatenate([[0], np.cumsum(w.run_pod_off[alive + 1] - w.run_pod_off[alive])]).astype(np.uint32)
    cn, co = (None, None) if cands is None else (cands[0][cands[1][p]:cands[1][p + 1]],
                                                np.array([0, cands[1][p + 1] - cands[1][p]], np.uint32))
    return PY.preempt_why(gpus, w.node_off, w.table, w.claims[c0:c1], np.array([0, c1 - c0], np.uint32), w.prio[p:p + 1],
                          w.run_claims[keep], rpo, w.run_prio[alive], w.run_out[keep], None, cn, co, w.flags_)


def pairs_of(w, p, cands):
    n_node = len(w.node_off) - 1
    return (p * n_node, (p + 1) * n_node) if cands is None else (int(cands[1][p]), int(cands[1][p + 1]))


def check(ctx, w, cands, oo, n_out, flags, name):
    cn, co = (None, None) if cands is None else cands
    n_pod, n_run = len(w.pod_off) - 1, len(w.run_pod_off) - 1
    w.flags_ = flags
    sample = np.random.default_rng(3).choice(n_pod, 3, replace=False).tolist() + [n_pod - 1]
    ctx.reset_inventory()
    st, why, claim, _, _ = ctx.preempt_why(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                                           None, cn, co, flags)
    ok = ctx.preempt(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co, 1,
                     flags)[0].tobytes() == st.tobytes()
    for p in sample:
        k0, k1 = pairs_of(w, p, cands)
        ref = one_pod(w, p, w.gpus, np.arange(n_run), cands)
        ok = ok and ref[0].tobytes() == st[k0:k1].tobytes() and ref[1].tobytes() == why[k0:k1].tobytes() and \
            [NONE if x == NONE else int(x) + int(w.pod_off[p]) for x in ref[2]] == claim[k0:k1].tolist()
    ctx.reset_inventory()
    got = ctx.preempt_place_why(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None,
                                cn, co, oo, n_out, flags)
    inv = ctx.get_inventory()
    ctx.reset_inventory()
    plain = ctx.preempt_place(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None,
                              cn, co, oo, n_out, flags)
    ok = ok and all(x.tobytes() == y.tobytes() for x, y in zip(plain, got[:4])) and \
        ctx.get_inventory().tobytes() == inv.tobytes()
    for p in sample:
        c0 = int(w.pod_off[p])
        pre = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims[:c0], w.pod_off[:p + 1], w.prio[:p], w.run_claims,
                               w.run_pod_off, w.run_prio, w.run_out, None, None if co is None else cn[:co[p]],
                               None if co is None else co[:p + 1], oo[:c0], n_out, flags)
        k0, k1 = pairs_of(w, p, cands)
        ref = one_pod(w, p, pre[4], np.flatnonzero(pre[3] == NONE), cands)
        ok = ok and ref[0].tobytes() == got[4][k0:k1].tobytes() and ref[1].tobytes() == got[5][k0:k1].tobytes() and \
            [NONE if x == NONE else int(x) + c0 for x in ref[2]] == got[6][k0:k1].tolist()
    print(f"oracle check {name}: {'ok' if ok else 'MISMATCH'} (§14 pairs FITS {int((st == 0).sum())}, EVICT "
          f"{int((st == 1).sum())}, NO {int((st == 2).sum())}; §15 pods EVICT {int((got[2] == 1).sum())})")
    if not ok:
        sys.exit(1)


def alternate(calls, setup):
    for fn in calls.values():
        setup(); fn()                                          # warm-up: buffers grown, modules loaded
    ts = {k: [] for k in calls}
    for _ in range(REPS):
        for k, fn in calls.items():
            setup()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); b.synchronize()
            ts[k].append(a.elapsed_time(b) * 1e3)
    base = statistics.median(next(iter(ts.values())))
    for k, v in ts.items():
        med = statistics.median(v)
        print(f"  {k:<20} median {med / 1e3:9.3f} ms (min {min(v) / 1e3:.3f}, max {max(v) / 1e3:.3f})  x{med / base:.2f}")


def main():
    torch.cuda.init()
    print(f"device (name, power limit, max SM clock): {card()}")
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
    print(f"{REPS} calls per case and call, alternating")
    with A.Context(device=0) as ctx:
        for wname, w in worlds.items():
            print(f"workload {wname}: {n_node} nodes x 8 GPUs, {len(w.run_pod_off) - 1} running pods, {n_pod} pending pods")
            placed = w.claims.copy(); placed["node"] = 0
            sl = R.claim_slots(placed, 1).astype(np.int64)
            oo, n_out = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32), int(sl.sum())
            ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
            for form, cc in (("dense", None), (f"{k} candidates", cands)):
                cn, co = (None, None) if cc is None else cc
                for flags in (0, A.F_EXHAUSTIVE):
                    name = f"{wname} {form}, flags {'EXHAUSTIVE' if flags else '0'}"
                    check(ctx, w, cc, oo, n_out, flags, name)
                    run = (w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co)
                    print(f"{name}: §14")
                    alternate({"preempt": lambda: ctx.preempt(w.claims, w.pod_off, w.prio, *run, 8, flags),
                               "preempt_why": lambda: ctx.preempt_why(w.claims, w.pod_off, w.prio, *run, flags)},
                              lambda: None)
                    print(f"{name}: §15")
                    alternate({"preempt_place": lambda: ctx.preempt_place(w.claims, w.pod_off, w.prio, *run, oo, n_out, flags),
                               "preempt_place_why": lambda: ctx.preempt_place_why(w.claims, w.pod_off, w.prio, *run, oo,
                                                                                  n_out, flags)},
                              ctx.reset_inventory)
    print(f"device after the run: {card()}")


if __name__ == "__main__":
    main()
