"""CPU suite: the oracle on Allocate problems at the record limits (tests/limit_problems.py): 16-slice shapes and starts up
to 15, nodes of up to 32 GPUs, 31-65 claims on a node (segment boundaries of the packing loops), co-location runs across
them, share counts and memory at 0xFFFF / 2^32 - 1.  The C oracle must equal the independent restatement (oracle/naive.py),
the tuned CPU port must equal the C oracle, and the spec's invariants must hold: placements come from the table and never
overlap, the inventory after the batch is the inventory before plus the successful results (a share count never passes
0xFFFF, free memory never goes below 0), and Deallocate restores it.  Pods Allocate and UnsuitableNodes, with and without
the exhaustive search, are checked the same way on pods cut from the same problems.  A fixed example set must keep
reaching every branch limit_problems.features() names."""
import os

import numpy as np
from hypothesis import HealthCheck, given, settings

import limit_problems as LP
from test_oracle_properties import _dicts
from test_pod_mode import _tbl

R = LP.R
N_EX = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))     # > 0: that many RANDOM examples instead of the fixed ones
N_FIXED = 60
# how often the fixed seeds 0 .. N_FIXED - 1 must reach each branch (each problem counts once per branch)
MIN_FEATURES = {"claims_31": 5, "claims_32": 5, "claims_33": 5, "claims_64": 5, "claims_65": 5, "node_17_32": 10,
                "fast3_ok": 3, "fast4_ok": 10, "fast_9_16_ok": 5, "fast_size9_row_max9": 3, "fast_small_row_junk_cell": 3,
                "start_ge8_ok": 10, "size16_ok": 3, "run_crosses_segment": 5, "run_crosses_segment_ok": 2, "run_32": 3,
                "run_cut_at_33": 3, "dead_shape_asked_in_later_segment": 10, "hetero_wide_and_small": 5,
                "hetero_placed_off_lane0_model": 5, "sh_segment": 10, "fast_sh_skips_share_ffff": 5,
                "share_reaches_ffff": 5, "shared_limit_eq_free_ok": 10, "shared_limit_max_ok": 5,
                "limit_max_ok_after_clean_sh_segment": 3}


def _naive_out(rows):
    return [tuple(int(v) for v in r) for r in rows]


def check_allocate(pb, oracle):
    from oracle import naive, tuned
    g, off, t, c, oo, n_out = pb.gpus, pb.node_off, pb.table, pb.claims, pb.out_off, pb.n_out
    n_node = pb.n_node
    out, after = oracle.allocate(g, off, t, c, oo, n_out)
    nout, nafter = naive.allocate(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in oo])
    assert _naive_out(out) == nout
    assert [(int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) for a in after] == \
           [(b["busy"], b["flags"], b["mem_free_mib"], b["share_cnt"]) for b in nafter]
    for th in (1, 4):
        tout, tafter = tuned.allocate(g, off, t, c, oo, n_out, threads=th)
        assert tout.tobytes() == out.tobytes() and tafter.tobytes() == after.tobytes(), th
    # invariants, in unbounded integers
    busy = g["busy"].astype(np.int64).copy()
    flags = g["flags"].astype(np.int64).copy()
    mem = g["mem_free_mib"].astype(np.int64).copy()
    share = g["share_cnt"].astype(np.int64).copy()
    slots = R.claim_slots(c, n_node)
    for i in range(len(c)):
        for k in range(int(slots[i])):
            o = out[int(oo[i]) + k]
            if o["status"] != R.ST_OK:
                assert o["gpu"] == R.GPU_NONE
                continue
            gi = int(o["gpu"])
            assert off[c[i]["node"]] <= gi < off[c[i]["node"] + 1]
            assert not flags[gi] & (R.GPU_UNAVAILABLE | R.GPU_FULL_ALLOCATED)
            if c[i]["kind"] == R.KIND_MIG:
                e = t[g["model"][gi], c[i]["profile"]]
                assert o["size"] == e["size"] and (int(e["start_mask"]) >> int(o["start"])) & 1
                assert int(o["start"]) + int(o["size"]) <= 16
                m = ((1 << int(o["size"])) - 1) << int(o["start"])
                assert busy[gi] & m == 0 and flags[gi] & R.GPU_MIG_ENABLED
                busy[gi] |= m
            elif c[i]["kind"] == R.KIND_GPU:
                assert not flags[gi] & R.GPU_MIG_ENABLED and share[gi] == 0
                flags[gi] |= R.GPU_FULL_ALLOCATED
            else:
                assert not flags[gi] & R.GPU_MIG_ENABLED
                mem[gi] -= int(c[i]["mem_limit_mib"])
                share[gi] += 1
    assert (mem >= 0).all() and (share <= 0xFFFF).all()                     # no wrap-around
    assert (after["busy"] == busy).all() and (after["flags"] == flags).all()
    assert (after["mem_free_mib"] == mem).all() and (after["share_cnt"] == share).all()
    back = oracle.deallocate(after, c, out, oo, n_node=n_node)
    assert back.tobytes() == g.tobytes()
    return out


def check_pods(pb, oracle, first=0, max_pairs=40):
    from oracle import naive
    c, pod_off, oo, n_out = LP.pods(pb, first)
    gd, offl, tbl = _dicts(pb.gpus), [int(x) for x in pb.node_off], _tbl(pb.table)
    n_node, n_pod = pb.n_node, len(pod_off) - 1
    for flags in (0, oracle.F_EXHAUSTIVE):
        out, after = oracle.allocate_pods(pb.gpus, pb.node_off, pb.table, c, pod_off, oo, n_out, flags)
        nout, nafter = naive.allocate_pods(gd, offl, tbl, _dicts(c), [int(x) for x in pod_off], bool(flags),
                                           [int(x) for x in oo])
        assert _naive_out(out) == nout, flags
        assert [(int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) for a in after] == \
               [(b["busy"], b["flags"], b["mem_free_mib"], b["share_cnt"]) for b in nafter]
        assert oracle.deallocate(after, c, out, oo, n_node=n_node).tobytes() == pb.gpus.tobytes()
        # UnsuitableNodes, dense: every pod against every node; the first max_pairs pairs against the restatement
        cn = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
        co = (np.arange(n_pod + 1) * n_node).astype(np.uint32)
        bits = oracle.unsuitable(pb.gpus, pb.node_off, pb.table, c, pod_off, cn, co, flags)
        got = np.unpackbits(bits, bitorder="little")[: n_pod * n_node]
        for k in range(min(len(got), max_pairs)):
            p, n = divmod(k, n_node)
            pod = [dict(x, node=n) for x in _dicts(c[pod_off[p]: pod_off[p + 1]])]
            if not pod:
                want = True
            elif len(pod) > R.MAX_POD:
                want = False
            elif flags:
                want = naive.eval_pod(naive._state(gd), offl[n], offl[n + 1], tbl, pod, n_node, True)[0]
            else:
                po, pn = R.out_offsets(c[pod_off[p]: pod_off[p + 1]].copy(), n_node)
                res, _ = naive.allocate(gd, offl, tbl, pod, [int(x) for x in po])
                want = all(r[4] == R.ST_OK for r in res[:pn])
            assert bool(got[k]) == want, (flags, p, n)


@settings(max_examples=N_EX or 40, deadline=None, suppress_health_check=list(HealthCheck), derandomize=N_EX == 0,
          database=None)
@given(LP.problems())
def test_oracle_agrees_with_naive_and_tuned_and_keeps_the_invariants(oracle, pb):
    check_allocate(pb, oracle)
    check_pods(pb, oracle)


def test_fixed_examples_reach_every_branch(oracle):
    """The seeded problems the GPU suite runs: oracle checks as above, and every branch of features() reached often
    enough that a change to the generator cannot quietly stop reaching one."""
    seen = {}
    for seed in range(N_FIXED):
        pb = LP.random_problem(seed)
        out = check_allocate(pb, oracle)
        if seed % 4 == 0:
            check_pods(pb, oracle, first=seed, max_pairs=12)
        for k in LP.features(pb, out):
            seen[k] = seen.get(k, 0) + 1
    low = {k: (seen.get(k, 0), n) for k, n in MIN_FEATURES.items() if seen.get(k, 0) < n}
    assert not low, f"branches reached too rarely (seen, needed): {low}"


def test_threaded_oracle_across_changing_thread_counts(oracle):
    """Regression: the multi-threaded oracle rebuilds its worker pool whenever a call's thread count changes (at most one
    thread per node).  Workers created after earlier batches started by taking the last batch as pending, so on a
    host with cores to spare they ran nodes of the next call twice (its first claims then found their own earlier
    placements and failed) and could report it done before it was.  The answer must not depend on the thread count."""
    for seed in range(N_FIXED):
        pb = LP.random_problem(seed)
        want, want_inv = oracle.allocate(pb.gpus, pb.node_off, pb.table, pb.claims, pb.out_off, pb.n_out)
        for th in (8, 3, 6, 2, 5):
            got, inv = oracle.allocate(pb.gpus, pb.node_off, pb.table, pb.claims, pb.out_off, pb.n_out, threads=th)
            assert got.tobytes() == want.tobytes() and inv.tobytes() == want_inv.tobytes(), (seed, th)
