"""CPU suite: spec §18 — why place pods put each pod where it did, or nowhere: every (pod, candidate) pair answered on
the state the pods before it left (W_p), with §13's own evaluation.

place_why_oracle.place_why (on the C oracle's place pods and its own §12 reasons over why_oracle's helpers) and place_why_naive (on
oracle/naive.py) share no code; the tests check that they agree, that the placement is §13's, and the consequences
§18 states: a pod goes to the node of its first OK pair, and with DRA_F_EXHAUSTIVE its pairs are §17's on the live
inventory after the pods before it."""
import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_place_pods import placed_offsets
from test_pod_capacity import R, _flat, problem
from test_pod_mode import _mig, _tbl

import place_oracle as P
import place_why_oracle as PW
import why_oracle as Y

NONE = 0xFFFFFFFF


def _pairs(pod_off, cn, co, n_node):
    """[(pod, node)] in pair order"""
    n_pod = len(pod_off) - 1
    if co is None:
        return [(p, n) for p in range(n_pod) for n in range(n_node)]
    return [(p, int(cn[k])) for p in range(n_pod) for k in range(int(co[p]), int(co[p + 1]))]


def _case(seed, with_off):
    g, off, t, c, pod_off, cands = problem(seed, n_node=4, n_run=20)
    cn, co = (None, None) if cands is None else _flat(cands)
    oo, n_out = placed_offsets(R, c, len(off) - 1) if with_off else (None, None)
    return g, off, t, c, pod_off, cands, cn, co, oo, n_out


def _out_tuples(out):
    return [(int(r["gpu"]), int(r["start"]), int(r["size"]), int(r["profile"]), int(r["status"])) for r in out]


@pytest.mark.parametrize("seed", range(16))
@pytest.mark.parametrize("flags", [0, Y.F_EXHAUSTIVE])
@pytest.mark.parametrize("with_off", [False, True])
def test_the_two_oracles_agree(seed, flags, with_off):
    g, off, t, c, pod_off, cands, cn, co, oo, n_out = _case(seed, with_off)
    a = PW.place_why(g, off, t, c, pod_off, cn, co, oo, n_out, flags)
    b = PW.place_why_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in pod_off],
                           None if cands is None else [[int(n) for n in x] for x in cands], bool(flags),
                           None if oo is None else [int(x) for x in oo])
    assert a[1].tolist() == b[1]
    assert a[3].tolist() == b[3] and a[4].tolist() == b[4]
    assert a[5].tolist() == b[5] and a[6].tolist() == b[6]
    assert [(int(x["busy"]), int(x["flags"]), int(x["mem_free_mib"]), int(x["share_cnt"])) for x in a[2]] == \
        [(x["busy"], x["flags"], x["mem_free_mib"], x["share_cnt"]) for x in b[2]]
    got = _out_tuples(a[0])
    for i, r in enumerate(b[0]):
        if r is not None:
            assert got[i] == tuple(int(v) for v in r), i


@pytest.mark.parametrize("seed", range(16))
@pytest.mark.parametrize("flags", [0, Y.F_EXHAUSTIVE])
@pytest.mark.parametrize("with_off", [False, True])
def test_placement_is_place_pods_and_consequences_hold(seed, flags, with_off):
    """out, pod_node and the state are §13's; consequence 1; each podWhy row counts the pod's pairs; the per-claim
    tallies add up; no SEARCH_LIMIT without the flag."""
    g, off, t, c, pod_off, cands, cn, co, oo, n_out = _case(seed, with_off)
    out, pod_node, after, why, claim, pod_why, blocks = PW.place_why(g, off, t, c, pod_off, cn, co, oo, n_out, flags)
    ref, ref_node, ref_after = P.place_pods(g, off, t, c, pod_off, cn, co, oo, n_out, flags)
    assert out.tobytes() == ref.tobytes() and pod_node.tobytes() == ref_node.tobytes()
    assert after.tobytes() == ref_after.tobytes()
    pairs = _pairs(pod_off, cn, co, len(off) - 1)
    assert len(pairs) == len(why) == len(claim)
    if not flags:
        assert Y.ST_SEARCH_LIMIT not in why.tolist()
    assert Y.ST_GROUP not in why.tolist()
    for p in range(len(pod_off) - 1):
        ks = [k for k, (q, _) in enumerate(pairs) if q == p]
        assert int(pod_why[p].sum()) == len(ks)
        assert pod_why[p].tolist() == np.bincount(why[ks].astype(np.int64), minlength=Y.WHY_N).tolist()
        cnt = int(pod_off[p + 1] - pod_off[p])
        if cnt == 0 or cnt > Y.MAX_POD:
            assert pod_node[p] == NONE
            continue
        oks = [pairs[k][1] for k in ks if why[k] == Y.ST_OK]
        assert pod_node[p] == (oks[0] if oks else NONE), p
    named = claim[claim != Y.WHY_CLAIM_NONE]
    assert blocks.tolist() == np.bincount(named.astype(np.int64), minlength=len(c)).tolist()
    assert ((why == Y.ST_OK) | (why == Y.WHY_NO_NODE) | (claim != Y.WHY_CLAIM_NONE) | (why == Y.ST_INVALID)).all()


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("with_off", [False, True])
def test_with_the_flag_pod_p_is_section_17_after_the_pods_before_it(seed, with_off):
    """Consequence 2: with DRA_F_EXHAUSTIVE, pod p's pairs are §17's with the flag on the inventory place pods leaves
    after pods 0..p-1 — except that §17 judges validity as if out_off were given."""
    g, off, t, c, pod_off, cands, cn, co, oo, n_out = _case(seed, with_off)
    why = PW.place_why(g, off, t, c, pod_off, cn, co, oo, n_out, Y.F_EXHAUSTIVE)[3]
    pairs = _pairs(pod_off, cn, co, len(off) - 1)
    n_pod = len(pod_off) - 1
    for p in range(n_pod):
        c0 = int(pod_off[p])
        pre_off = pod_off[: p + 1]
        pre_co = None if co is None else co[: p + 1]
        pre_oo = None if oo is None else oo[:c0]
        _, _, live = P.place_pods(g, off, t, c[:c0], pre_off, cn, pre_co, pre_oo, n_out if with_off else c0,
                                  Y.F_EXHAUSTIVE)
        one_off = np.array([0, int(pod_off[p + 1]) - c0], np.uint32)
        one_cn = None if co is None else cn[co[p]:co[p + 1]]
        one_co = None if co is None else np.array([0, int(co[p + 1] - co[p])], np.uint32)
        w17 = Y.why(live, off, t, c[c0:int(pod_off[p + 1])], one_off, one_cn, one_co, Y.F_EXHAUSTIVE)[0]
        ks = [k for k, (q, _) in enumerate(pairs) if q == p]
        invalid_by_slot_mode = not with_off and any(
            x["kind"] == Y.KIND_GPU and x["count"] != 1 for x in c[c0:int(pod_off[p + 1])])
        if not invalid_by_slot_mode:
            assert why[ks].tolist() == w17.tolist(), p


def test_the_pod_that_lost_the_last_slot():
    """Two pods need the last 3g slot of the only node: the second is NO_CAPACITY there (the state it met), while §17
    on the snapshot says OK."""
    g, off = R.make_inventory([1], mig=True)
    g["busy"][0] = 0b1111                       # 4g taken: one 3g slot left (starts 4 only)
    t = R.default_table()
    c = _mig(R, [R.GI_3_SLICE, R.GI_3_SLICE])
    pod_off = np.array([0, 1, 2], np.uint32)
    cn, co = _flat([[0], [0]])
    for flags in (0, Y.F_EXHAUSTIVE):
        out, pod_node, _, why, claim, pod_why, _ = PW.place_why(g, off, t, c, pod_off, cn, co, flags=flags)
        assert pod_node.tolist() == [0, NONE]
        assert why.tolist() == [Y.ST_OK, Y.ST_NO_CAPACITY] and claim.tolist() == [Y.WHY_CLAIM_NONE, 1]
        assert pod_why[1, Y.ST_NO_CAPACITY] == 1
        snap = Y.why(g, off, t, c, pod_off, cn, co, flags)[0]
        assert snap.tolist() == [Y.ST_OK, Y.ST_OK]


def test_later_pairs_are_dry_runs_and_the_chosen_node_is_ok():
    """Pairs after the one that took the pod are answered on W_p: a later listing of the chosen node is OK, and the
    pod's own placement does not make another node look full."""
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    c = _mig(R, [R.GI_7_SLICE])
    pod_off = np.array([0, 1], np.uint32)
    cn, co = _flat([[0, 1, 0, 7]])
    _, pod_node, _, why, claim, _, _ = PW.place_why(g, off, t, c, pod_off, cn, co, flags=0)
    assert pod_node.tolist() == [0]
    assert why.tolist() == [Y.ST_OK, Y.ST_OK, Y.ST_OK, Y.WHY_NO_NODE]


def test_gpu_claim_of_count_two_is_invalid_without_out_off():
    g, off = R.make_inventory([4], mig=False)
    t = R.default_table()
    c = np.zeros(1, R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_GPU, 2
    pod_off = np.array([0, 1], np.uint32)
    oo, n_out = placed_offsets(R, c, 1)
    w = PW.place_why(g, off, t, c, pod_off, flags=Y.F_EXHAUSTIVE)
    assert w[3].tolist() == [Y.ST_INVALID] and w[4].tolist() == [0] and w[1].tolist() == [NONE]
    w = PW.place_why(g, off, t, c, pod_off, out_off=oo, n_out=n_out, flags=Y.F_EXHAUSTIVE)
    assert w[3].tolist() == [Y.ST_OK] and w[1].tolist() == [0]


@pytest.mark.parametrize("seed", range(8))
def test_with_backtracking_and_out_off_the_reasons_are_section_17s(seed):
    """pair_reason and naive_pod_reason with backtracking and out_off's validity are §17's exhaustive answers
    (why_oracle's _pair and _naive_pod) on the same state, pair for pair."""
    import copy

    from oracle import naive as N
    g, off, t, c, pod_off, cands, cn, co, _, _ = _case(seed, False)
    n_node = len(off) - 1
    gd, td, cd = _dicts(g), _tbl(t), _dicts(c)
    for p, n in _pairs(pod_off, cn, co, n_node):
        c0, c1 = int(pod_off[p]), int(pod_off[p + 1])
        assert PW.pair_reason(g, off, t, c, c0, c1, n, None, None, True, True) == \
            Y._pair(g, off, t, c, c0, c1, n, Y.F_EXHAUSTIVE, None, None)
        if n < n_node:
            W = N._state(gd)[int(off[n]):int(off[n + 1])]
            pod = [dict(x, node=n) for x in cd[c0:c1]]
            assert PW.naive_pod_reason(N, copy.deepcopy(W), td, pod, n_node, True, True) == \
                Y._naive_pod(N, copy.deepcopy(W), td, pod, n_node)
