"""Spec §17 on the CPU: the reasons oracle (tests/why_oracle.py) against the bit oracles of §8 / §12 and §16's pod
capacity, its tallies, and the meaning of the search depth d."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from test_pod_capacity import R, _flat, problem

import capacity_oracle as K
import why_oracle as Y
from oracle import oracle as O


def _all_cands(n_pod, n_node):
    return [list(range(n_node)) for _ in range(n_pod)]


def _bits(g, off, t, c, pod_off, cands, flags):
    cn, co = _flat(cands)
    b = O.unsuitable(g, off, t, c, pod_off, cn, co, flags)
    return np.unpackbits(np.asarray(b, np.uint8), bitorder="little")[: int(co[-1])].astype(bool)


@pytest.mark.parametrize("flags", [0, Y.F_EXHAUSTIVE])
@pytest.mark.parametrize("seed", range(6))
def test_ok_is_the_unsuitable_bit_and_tallies_add_up(seed, flags):
    g, off, t, c, pod_off, cands = problem(7100 + seed, n_node=5, n_run=30)
    n_node, n_pod = len(off) - 1, len(pod_off) - 1
    cn, co = (None, None) if cands is None else _flat(cands)
    why, claim, pod_why, blocks = Y.why(g, off, t, c, pod_off, cn, co, flags)
    full = cands if cands is not None else _all_cands(n_pod, n_node)
    assert ((why == Y.ST_OK) == _bits(g, off, t, c, pod_off, full, flags)).all()
    assert ((claim == Y.WHY_CLAIM_NONE) >= (why == Y.ST_OK)).all()
    counts = [len(x) for x in full]
    assert pod_why.sum(axis=1).tolist() == counts
    assert int(blocks.sum()) == int((claim != Y.WHY_CLAIM_NONE).sum())
    # every blocking claim lies in its own pod
    k = 0
    for p, n in enumerate(counts):
        for _ in range(n):
            if claim[k] != Y.WHY_CLAIM_NONE:
                assert pod_off[p] <= claim[k] < pod_off[p + 1]
            k += 1
    if cands is not None:
        stray = np.array([x >= n_node for x in cn[: int(co[-1])]], bool)
        assert ((why == Y.WHY_NO_NODE) == stray).all()


@pytest.mark.parametrize("seed", range(4))
def test_exhaustive_ok_is_capacity_at_least_one(seed):
    g, off, t, c, pod_off, cands = problem(7200 + seed, n_node=5, n_run=30)
    cn, co = (None, None) if cands is None else _flat(cands)
    why, _, _, _ = Y.why(g, off, t, c, pod_off, cn, co, Y.F_EXHAUSTIVE)
    copies = K.capacity(g, off, t, c, pod_off, cn, co, 1, K.F_EXHAUSTIVE)[0]
    assert ((why == Y.ST_OK) == (copies >= 1)).all()


def test_search_depth_is_the_deepest_placeable_prefix():
    """With the flag, a pair failing with POD at MIG claim m (the level d): the pod cut before m (its other claims and
    the MIG claims before m) fits the node, and the pod cut after m does not — the search held d levels and never d + 1."""
    seen = 0
    for seed in range(40):
        seen += _depth_cases(seed)
    assert seen


def _depth_cases(seed):
    g, off, t, c, pod_off, _ = problem(7300 + seed, n_node=4, n_run=60)
    n_node, n_pod = len(off) - 1, len(pod_off) - 1
    why, claim, _, _ = Y.why(g, off, t, c, pod_off, None, None, Y.F_EXHAUSTIVE)
    seen = 0
    for p in range(n_pod):
        for n in range(n_node):
            k = p * n_node + n
            if why[k] != Y.ST_POD:
                continue
            m = int(claim[k])
            assert c[m]["kind"] == Y.KIND_MIG
            pod = c[pod_off[p]:pod_off[p + 1]]
            keep = [i for i in range(len(pod)) if pod[i]["kind"] != Y.KIND_MIG or pod_off[p] + i < m]
            for cut, fits in ((keep, True), (keep + [m - pod_off[p]], False)):
                sub = pod[sorted(cut)]
                bit = _bits(g, off, t, sub, np.array([0, len(sub)], np.uint32), [[n]], Y.F_EXHAUSTIVE)[0]
                assert bool(bit) == fits, (seed, p, n, m)
            seen += 1
    return seen


def test_in_order_walk_names_the_first_failing_slot():
    """Without the flag: a GPU claim that cannot fit, then a MIG claim that is invalid — the GPU claim blocks; a pod
    naming a node past the inventory is NO_NODE; an empty pod is OK everywhere."""
    t = R.default_table()
    g = np.zeros(2, O.GPU_DTYPE)
    g["flags"] = 1                                   # both GPUs MIG-enabled: a full-GPU claim finds no GPU
    off = np.array([0, 2], np.uint32)
    c = np.zeros(2, O.CLAIM_DTYPE)
    c[0]["kind"], c[0]["count"] = Y.KIND_GPU, 1
    c[1]["kind"], c[1]["profile"] = Y.KIND_MIG, 99
    pod_off = np.array([0, 2, 2], np.uint32)
    cn, co = np.array([0, 5, 0], np.uint32), np.array([0, 2, 3], np.uint32)
    why, claim, pod_why, blocks = Y.why(g, off, t, c, pod_off, cn, co, 0)
    assert why.tolist() == [Y.ST_NO_CAPACITY, Y.WHY_NO_NODE, Y.ST_OK]
    assert claim.tolist() == [0, Y.WHY_CLAIM_NONE, Y.WHY_CLAIM_NONE]
    assert blocks.tolist() == [1, 0]
    assert pod_why[0, Y.ST_NO_CAPACITY] == 1 and pod_why[0, Y.WHY_NO_NODE] == 1 and pod_why[1, Y.ST_OK] == 1
    # with the flag the invalid claim comes first (step 1)
    why, claim, _, _ = Y.why(g, off, t, c, pod_off, cn, co, Y.F_EXHAUSTIVE)
    assert why.tolist() == [Y.ST_INVALID, Y.WHY_NO_NODE, Y.ST_OK] and claim.tolist()[0] == 1


def test_pods_over_32_claims_are_invalid_with_the_flag_only():
    t = R.default_table()
    g = np.zeros(1, O.GPU_DTYPE)
    off = np.array([0, 1], np.uint32)
    c = np.zeros(33, O.CLAIM_DTYPE)
    c["kind"] = Y.KIND_SHARED
    pod_off = np.array([0, 33], np.uint32)
    assert Y.why(g, off, t, c, pod_off, None, None, 0)[0].tolist() == [Y.ST_OK]
    why, claim, _, _ = Y.why(g, off, t, c, pod_off, None, None, Y.F_EXHAUSTIVE)
    assert why.tolist() == [Y.ST_INVALID] and claim.tolist() == [Y.WHY_CLAIM_NONE]


@settings(max_examples=40, deadline=None, suppress_health_check=list(HealthCheck))
@given(seed=st.integers(0, 2**31 - 1), exhaustive=st.booleans())
def test_the_two_oracles_agree(seed, exhaustive):
    """The oracle on the C Allocate and the restatement on oracle/naive.py, on the pod-capacity generator's problems
    (every claim kind, groups, invalid claims, 0 to 33 claims, strays, the dense form; no selectors)."""
    from test_oracle_properties import _dicts
    from test_pod_mode import _tbl
    g, off, t, c, pod_off, cands = problem(seed, n_node=4, n_run=20)
    cn, co = (None, None) if cands is None else _flat(cands)
    a = Y.why(g, off, t, c, pod_off, cn, co, Y.F_EXHAUSTIVE if exhaustive else 0)
    b = Y.why_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in pod_off],
                    None if cands is None else [[int(n) for n in x] for x in cands], exhaustive)
    assert a[0].tolist() == b[0] and a[1].tolist() == b[1]
    assert a[2].tolist() == b[2] and a[3].tolist() == b[3]
