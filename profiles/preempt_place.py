"""Preempt and place (spec §15) timings on one GPU: dra_preempt_place_batch on the worlds of profiles/preempt.py, every
case checked against the CPU oracle before anything is timed, against the host loop it replaces.  Workloads:
  cfg2-sized    125 nodes x 8 MIG GPUs, ~90 % taken by 1g and 2g running pods at priorities 0..999, 1,000 pending 3g, 7g
                and 2x3g pods at priority 1000; dense and 16 random candidates per pod, each with and without
                DRA_F_EXHAUSTIVE;
  SHARED-heavy  125 non-MIG nodes x 8 GPUs carrying up to 40 time-slicing / MPS pods each, 1,000 pending 4-GPU pods.
The call's time is the median (min, max) of repeated calls, CUDA events around the host-buffer call, the live inventory
reset before each.  The host loop is, per pod: dra_preempt_batch with that pod against the running pods not evicted yet,
dra_deallocate_batch of its victims, dra_allocate_pods_batch on the chosen node — three synchronising calls, with the
host-side bookkeeping between them; it is timed whole, on the host clock, and its result is checked against the call's.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))                # the CPU oracle of spec §15 (test infrastructure)
pkg = importlib.import_module("k8s-dra-driver_b200")
import preempt_place_oracle as PP  # noqa: E402

A, S, R = pkg.api, pkg.synth, pkg.records
REPS = int(os.environ.get("PREEMPT_PLACE_REPS", "5"))
LOOP_REPS = int(os.environ.get("PREEMPT_PLACE_LOOP_REPS", "2"))
NONE = 0xFFFFFFFF


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, setup):
    setup(); fn()                                              # warm-up: buffers grown, modules loaded
    ts = []
    for _ in range(REPS):
        setup()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


def host_loop(ctx, w, cands, oo, n_out, flags):
    """the per-pod loop on the device; returns (out of the placed pods' slots, mask of them, pod_node, evicted_by)"""
    n_node, n_run = len(w.node_off) - 1, len(w.run_pod_off) - 1
    ev = np.full(n_run, NONE, np.uint32)
    out = np.zeros(n_out, R.OUT_DTYPE)
    placed = np.zeros(n_out, bool)
    claim_of = np.repeat(np.arange(n_run), np.diff(w.run_pod_off))
    nodes = np.full(len(w.pod_off) - 1, NONE, np.uint32)
    for p in range(len(w.pod_off) - 1):
        c0, c1 = int(w.pod_off[p]), int(w.pod_off[p + 1])
        alive = np.flatnonzero(ev == NONE)
        keep = ev[claim_of] == NONE
        rpo = np.concatenate([[0], np.cumsum(w.run_pod_off[alive + 1] - w.run_pod_off[alive])]).astype(np.uint32)
        cn, co = (None, None) if cands is None else (cands[0][cands[1][p]: cands[1][p + 1]],
                                                    np.array([0, cands[1][p + 1] - cands[1][p]], np.uint32))
        _, _, pn, ps, nv, vic = ctx.preempt(w.claims[c0:c1], np.array([0, c1 - c0], np.uint32), w.prio[p:p + 1],
                                            w.run_claims[keep], rpo, w.run_prio[alive], w.run_out[keep], None, cn, co,
                                            max(len(alive), 1), flags)
        nodes[p] = pn[0]
        victims = alive[vic[0][: nv[0]]]
        if len(victims):
            ev[victims] = p
            vk = np.isin(claim_of, victims)
            ctx.deallocate(w.run_claims[vk], w.run_out[vk])
        if pn[0] != NONE and c1 > c0:
            pod = w.claims[c0:c1].copy()
            pod["node"] = pn[0]
            po_ = ctx.allocate_pods(pod, np.array([0, c1 - c0], np.uint32), oo[c0:c1] - oo[c0], n_out - int(oo[c0]), flags)
            n = int(R.claim_slots(pod, n_node).sum())
            out[oo[c0]: oo[c0] + n] = po_[:n]
            placed[oo[c0]: oo[c0] + n] = True
    return out, placed, nodes, ev


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
            placed_c = w.claims.copy(); placed_c["node"] = 0
            sl = R.claim_slots(placed_c, 1).astype(np.int64)
            oo, n_out = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32), int(sl.sum())
            ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
            for form, cc in (("dense", None), (f"{k} candidates", cands)):
                cn, co = (None, None) if cc is None else cc
                for flags in (0, A.F_EXHAUSTIVE):
                    args = (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, None, cn, co,
                            oo, n_out, flags)
                    ctx.reset_inventory()
                    got = ctx.preempt_place(*args)
                    inv = ctx.get_inventory()
                    t0 = time.perf_counter()
                    ref = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims,
                                           w.run_pod_off, w.run_prio, w.run_out, None, cn, co, oo, n_out,
                                           PP.F_EXHAUSTIVE if flags else 0)
                    t_cpu = time.perf_counter() - t0
                    ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and inv.tobytes() == ref[4].tobytes()
                    what = f"{wname} {form}, flags {'EXHAUSTIVE' if flags else '0'}"
                    print(f"oracle check {what}: {'ok' if ok else 'MISMATCH'} (pods FITS {int((got[2] == 0).sum())}, "
                          f"EVICT {int((got[2] == 1).sum())}, other {int((got[2] > 1).sum())}; "
                          f"{int((got[3] != NONE).sum())} running pods evicted)")
                    if not ok:
                        sys.exit(1)
                    med, lo, hi = timed(lambda: ctx.preempt_place(*args), ctx.reset_inventory)
                    print(f"  preempt_place: median {med / 1e3:9.2f} ms (min {lo / 1e3:.2f}, max {hi / 1e3:.2f}); "
                          f"CPU oracle, one thread: {t_cpu * 1e3:.0f} ms")
                    ts = []
                    for _ in range(LOOP_REPS):
                        ctx.reset_inventory()
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        lout, lmask, lnode, lev = host_loop(ctx, w, cc, oo, n_out, flags)
                        ts.append(time.perf_counter() - t0)
                        same = lev.tobytes() == got[3].tobytes() and lnode.tobytes() == got[1].tobytes() and \
                            lout[lmask].tobytes() == got[0][lmask].tobytes() and ctx.get_inventory().tobytes() == inv.tobytes()
                        if not same:
                            print("  host loop: MISMATCH with the call")
                            sys.exit(1)
                    print(f"  host loop ({n_pod} x 3 calls): median {statistics.median(ts) * 1e3:9.2f} ms "
                          f"(min {min(ts) * 1e3:.2f}, max {max(ts) * 1e3:.2f}); same result as the call")


if __name__ == "__main__":
    main()
