"""CPU suite: spec §13 — place a batch of pods on the first candidate node each one fits, given what the pods before it
took (the batched form of the classic controller's pending allocations, SURVEY App. A).

The C oracle (tests/place_oracle.c, on oracle/dra_oracle.c's pod evaluation) and the pure-Python restatement
(place_oracle.place_pods_naive, on oracle/naive.py's) share no code, so agreement between them pins the sequential rule."""
import numpy as np
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl, pod_problems

import place_oracle as P

NONE = 0xFFFFFFFF


def placed_offsets(R, claims, n_node):
    """out_off / n_out with slots counted as if every claim named a node of the inventory (spec §13)."""
    c = claims.copy()
    c["node"] = 0
    return R.out_offsets(c, max(n_node, 1))


def _flat(cands):
    off = np.zeros(len(cands) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in cands])
    nodes = np.array([n for x in cands for n in x], dtype=np.uint32)
    return nodes, off


def test_two_pods_two_nodes(pkg, oracle):
    """UnsuitableNodes judges both pods on one snapshot and says node 0 fits both; placing them one after the other
    sends the second to node 1."""
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    c = _mig(R, [R.GI_7_SLICE, R.GI_7_SLICE])
    pod_off = np.array([0, 1, 2], np.uint32)
    cn, co = _flat([[0, 1], [0, 1]])
    bits = oracle.unsuitable(g, off, t, c, pod_off, cn, co)
    assert bits[0] & 0xF == 0xF                                            # all four pairs "suitable"
    for cand in ((cn, co), (None, None)):
        out, pod_node, after = P.place_pods(g, off, t, c, pod_off, *cand)
        assert list(pod_node) == [0, 1]
        assert list(out["status"]) == [R.ST_OK, R.ST_OK] and list(out["gpu"]) == [0, 1]
        assert list(after["busy"]) == [0xFF, 0xFF]
    # the same through allocate_pods when the caller picks node 0 for both: the second fails
    c2 = c.copy(); c2["node"] = 0
    out, _ = oracle.allocate_pods(g, off, t, c2, pod_off)
    assert list(out["status"]) == [R.ST_OK, R.ST_POD]


def test_single_candidate_equals_allocate_pods(pkg, oracle):
    for seed, width in ((0, 8), (1, 16), (2, 32)):
        w, pod_off = pkg.synth.pods(1500, 12, seed, gpus_per_node=width)
        first = w.claims["node"][pod_off[:-1]]
        cn, co = first.astype(np.uint32), np.arange(len(pod_off), dtype=np.uint32)
        for flags in (0, oracle.F_EXHAUSTIVE):
            ref, inv = oracle.allocate_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, flags=flags)
            out, pod_node, after = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, flags=flags)
            assert out.tobytes() == ref.tobytes() and after.tobytes() == inv.tobytes()
            ok = np.array([ref["status"][pod_off[p]] == 0 for p in range(len(pod_off) - 1)])
            assert (pod_node[ok] == first[ok]).all() and (pod_node[~ok] == NONE).all()


def test_dense_equals_ascending_lists(pkg, oracle):
    w, pod_off = pkg.synth.pods(2000, 10, 3)
    n_pod, n_node = len(pod_off) - 1, w.n_node
    cn = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
    co = (np.arange(n_pod + 1) * n_node).astype(np.uint32)
    for flags in (0, oracle.F_EXHAUSTIVE):
        a = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, flags=flags)
        b = P.place_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, flags=flags)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        assert (a[1] != NONE).any() and (a[1] == NONE).any()


def test_search_limit_survives_a_later_pod_failure(pkg, oracle):
    """7 x 1g + 7g: the exhaustive search runs out of budget on the empty GPU of node 0; node 1 is full, where the
    pre-check fails the pod with POD.  The pod's records keep SEARCH_LIMIT."""
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    g["busy"][1] = 0xFF
    t = R.default_table()
    c = _mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])
    pod_off = np.array([0, 8], np.uint32)
    cn, co = _flat([[0, 1]])
    out, pod_node, after = P.place_pods(g, off, t, c, pod_off, cn, co, flags=oracle.F_EXHAUSTIVE)
    assert set(out["status"]) == {R.ST_SEARCH_LIMIT} and list(pod_node) == [NONE]
    assert after.tobytes() == g.tobytes()
    out, _, _ = P.place_pods(g, off, t, c, pod_off, cn, co)
    assert set(out["status"]) == {R.ST_POD}
    cn, co = _flat([[1, 0]])                                               # order of the candidates does not matter here
    out, _, _ = P.place_pods(g, off, t, c, pod_off, cn, co, flags=oracle.F_EXHAUSTIVE)
    assert set(out["status"]) == {R.ST_SEARCH_LIMIT}


def test_malformed_and_empty_pods(pkg, oracle):
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    # pods: [33 claims] [] [1g, invalid profile, 1g] [1g] [1g with no usable candidate] [GPU count 3]
    c = np.concatenate([_mig(R, [0] * 33), _mig(R, [0, 200, 0]), _mig(R, [0]), _mig(R, [0]),
                        np.zeros(1, dtype=R.CLAIM_DTYPE)])
    c[-1]["kind"], c[-1]["count"] = R.KIND_GPU, 3
    c["node"] = 99                                                         # ignored: never read, never written
    pod_off = np.array([0, 33, 33, 36, 37, 38, 39], np.uint32)
    cn, co = _flat([[0], [0], [0, 1], [5, 1, 1], [7, 9], [0, 1]])
    out_off, n_out = placed_offsets(R, c, 2)
    assert n_out == 33 + 3 + 1 + 1 + 3
    out, pod_node, after = P.place_pods(g, off, t, c, pod_off, cn, co, out_off, n_out)
    st_ = out["status"]
    assert set(st_[:33]) == {R.ST_INVALID}
    assert list(st_[33:36]) == [R.ST_POD, R.ST_INVALID, R.ST_POD]
    assert st_[36] == R.ST_OK and out["gpu"][36] == 1                      # node 5 is skipped, node 1 taken
    assert st_[37] == R.ST_POD and out["gpu"][37] == NONE                 # no candidate names a node: POD
    assert list(st_[38:41]) == [R.ST_POD] * 3                              # three slots, no non-MIG GPU anywhere
    assert list(pod_node) == [NONE, NONE, NONE, 1, NONE, NONE]
    assert int(after["busy"][1]) == 1 and int(after["busy"][0]) == 0
    # without out_off a GPU claim of count 3 is INVALID, with one slot
    out, _, _ = P.place_pods(g, off, t, c[:38], pod_off[:-1], cn[:co[-2]], co[:-1])
    assert out["status"][36] == R.ST_OK


def test_bad_arguments_leave_nothing_changed(pkg, oracle):
    import pytest
    R = pkg.records
    g, off = R.make_inventory([1, 1], mig=True)
    t = R.default_table()
    c = _mig(R, [0, 0])
    pod_off = np.array([0, 1, 2], np.uint32)
    with pytest.raises(ValueError):                                        # slot outside n_out
        P.place_pods(g, off, t, c, pod_off, out_off=np.array([0, 1], np.uint32), n_out=1)
    with pytest.raises(ValueError):                                        # pod_off not monotone
        P.place_pods(g, off, t, c, np.array([0, 2, 1, 2], np.uint32))
    with pytest.raises(ValueError):                                        # pod_off does not span the claims
        P.place_pods(g, off, t, c, np.array([0, 1], np.uint32))
    with pytest.raises(ValueError):                                        # cand_off not monotone
        P.place_pods(g, off, t, c, pod_off, np.array([0, 1], np.uint32), np.array([0, 2, 1], np.uint32))
    with pytest.raises(ValueError):                                        # unknown flags
        P.place_pods(g, off, t, c, pod_off, flags=0x100)


@st.composite
def place_problems(draw):
    g, off, t, c, pod_off, out_off, n_out = draw(pod_problems())
    n_node, n_pod = len(off) - 1, len(pod_off) - 1
    cands = []
    for _ in range(n_pod):
        k = draw(st.integers(0, 5))
        cands.append([draw(st.one_of(st.integers(0, max(n_node - 1, 0)), st.integers(0, n_node + 2)))
                      for _ in range(k)])
        if cands[-1] and draw(st.booleans()):
            cands[-1].append(cands[-1][0])                                 # a repeat
    return g, off, t, c, pod_off, cands, draw(st.booleans())


@settings(max_examples=300, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(place_problems(), st.booleans())
def test_place_oracle_agrees_with_naive(pkg, oracle, prob, exhaustive):
    R = pkg.records
    g, off, t, c, pod_off, cands, dense = prob
    n_node = len(off) - 1
    flags = oracle.F_EXHAUSTIVE if exhaustive else 0
    out_off, n_out = placed_offsets(R, c, n_node)
    cn, co = (None, None) if dense else _flat(cands)
    out, pod_node, after = P.place_pods(g, off, t, c, pod_off, cn, co, out_off, n_out, flags)
    nout, nnode, nafter = P.place_pods_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c),
                                           [int(x) for x in pod_off], None if dense else cands, exhaustive,
                                           [int(x) for x in out_off])
    assert [tuple(int(v) for v in r) for r in out][:len(nout)] == nout
    assert [int(x) for x in pod_node] == nnode
    for a, b in zip(after, nafter):
        assert (int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) == \
               (b["busy"], b["flags"], b["mem_free_mib"], b["share_cnt"])
    # a placed pod's devices lie on its node; Deallocate of the result (claims naming their node) restores the start
    placed = c.copy()
    for p in range(len(pod_off) - 1):
        placed["node"][pod_off[p]: pod_off[p + 1]] = pod_node[p] if pod_node[p] != NONE else 0
        for i in range(pod_off[p], pod_off[p + 1]):
            o = out[int(out_off[i])]
            if o["status"] == 0:
                assert pod_node[p] != NONE and off[pod_node[p]] <= o["gpu"] < off[pod_node[p] + 1]
    if n_node:
        back = oracle.deallocate(after, placed, out, out_off, n_node=n_node)
        assert back.tobytes() == g.tobytes()
