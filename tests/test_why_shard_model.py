"""CPU suite: spec §17 "Sharded form" — why splitting the pairs over the ranks gives the single-inventory reasons.

The sharded reasons call lets the rank whose node range holds a pair's candidate node judge that pair on its own copy of
the inventory, answers a candidate naming no node in place, and takes each pod's and each claim's tallies over the merged
pairs.  This model does exactly that with the CPU oracle (tests/why_oracle.py): every rank holds a DIVERGED copy (the
world's state on its own range, something else outside it), answers only its own pairs as a candidate list of its own,
and the merged result must equal the oracle on the world's state for any partition of the nodes, empty ranges
included."""
import numpy as np
import pytest

from test_capacity_shard_model import bounds_of, diverged, pairs, pristine
from test_pod_capacity import R, _flat, problem

import why_oracle as Y
from oracle import oracle as O

NONE = 0xFFFFFFFF
NAMES = ("pair_why", "pair_claim", "pod_why", "claim_blocks")


def sharded(copies, off, t, claims, pod_off, cn, co, flags, bounds, attrs=None, sels=None):
    """The sharded call's answer: rank r judges, on copies[r], only the pairs whose node lies in its range (its window, as
    a candidate list of its own); strays are NO_NODE with no claim; the tallies are taken over the merged pairs."""
    n_node, n_pod = len(off) - 1, len(pod_off) - 1
    pod, node = pairs(pod_off, cn, co, n_node)
    n_pair = len(node)
    why = np.full(n_pair, Y.WHY_NO_NODE, np.uint8)
    blk = np.full(n_pair, Y.WHY_CLAIM_NONE, np.uint32)
    owner = np.searchsorted(np.asarray(bounds), node, side="right") - 1
    for r in range(len(bounds) - 1):
        mine = np.flatnonzero((node < n_node) & (owner == r))
        if len(mine) == 0:
            continue
        sub_off = np.zeros(n_pod + 1, np.uint32)
        sub_off[1:] = np.cumsum(np.bincount(pod[mine], minlength=n_pod))
        w, c, _, _ = Y.why(copies[r], off, t, claims, pod_off, node[mine].astype(np.uint32), sub_off, flags, attrs, sels)
        why[mine], blk[mine] = w, c
    pod_why = np.zeros((n_pod, Y.WHY_N), np.uint32)
    np.add.at(pod_why, (pod, why.astype(np.int64)), 1)
    blocks = np.zeros(len(claims), np.uint32)
    named = blk != Y.WHY_CLAIM_NONE
    np.add.at(blocks, blk[named].astype(np.int64), 1)
    return why, blk, pod_why, blocks


def check(state, copies, off, t, claims, pod_off, cn, co, flags, bounds, what, attrs=None, sels=None):
    ref = Y.why(state, off, t, claims, pod_off, cn, co, flags, attrs, sels)
    got = sharded(copies, off, t, claims, pod_off, cn, co, flags, bounds, attrs, sels)
    for name, x, y in zip(NAMES, got, ref):
        assert x.tobytes() == np.ascontiguousarray(y, x.dtype).reshape(x.shape).tobytes(), f"{what}: {name}"
    return ref


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
def test_any_partition_gives_the_single_inventory_answer(world):
    """Random problems (strays, duplicates, empty, over-32-claim and INVALID pods, dense and candidate forms), random
    partitions, each rank's copy wrong outside its own range: the merged answer is the oracle's on the world's state."""
    rng = np.random.default_rng(world)
    differs, reasons, big = 0, set(), False
    for seed in range(12):
        n_node = 5 + seed % 6
        g, off, t, c, pod_off, cands = problem(700 * world + seed, n_node=n_node)
        g0 = pristine(700 * world + seed, n_node)
        full = g.copy()
        full["busy"] = 0xFFFF
        cn, co = (None, None) if cands is None else _flat(cands)
        big |= bool((np.diff(pod_off.astype(np.int64)) > Y.MAX_POD).any())
        bounds = bounds_of(rng, n_node, world)
        copies = [diverged(g, off, bounds, r, (g0, full)[r % 2]) for r in range(world)]
        for flags in (0, Y.F_EXHAUSTIVE):
            ref = check(g, copies, off, t, c, pod_off, cn, co, flags, bounds, f"w{world} seed {seed} f{flags}")
            reasons |= set(ref[0].tolist())
            if world > 1:
                alone = Y.why(copies[0], off, t, c, pod_off, cn, co, flags)
                differs += alone[0].tobytes() != ref[0].tobytes()
    assert {Y.ST_OK, Y.ST_INVALID, Y.ST_NO_CAPACITY, Y.WHY_NO_NODE} <= reasons, reasons
    assert big, "no pod of more than 32 claims"
    assert world == 1 or differs > 0                         # the diverged copies matter: one rank alone is wrong


@pytest.mark.parametrize("world", [2, 3])
def test_search_limit_and_strays_across_ranks(world):
    """A pod whose exhaustive search runs out of its budget (SEARCH_LIMIT, blocked by the MIG claim of level d), a
    selector no GPU passes (BAD_PROFILE), an INVALID claim, an empty pod, strays and duplicates, over ranges that split the
    two nodes every way; the tallies count each blocking claim once per pair across the ranks."""
    t = R.default_table()
    g = np.zeros(8, O.GPU_DTYPE)
    g["flags"], g["node"] = 1, np.repeat([0, 1], 4)
    off = np.array([0, 4, 8], np.uint32)
    attrs = np.zeros(8, R.ATTR_DTYPE)
    attrs["index"] = np.arange(8) % 4
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 0)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GT, 9))])
    small = int(np.flatnonzero(t[0]["size"] == 1)[0])
    c = np.zeros(33, O.CLAIM_DTYPE)
    c["kind"] = Y.KIND_MIG
    c["profile"] = small
    c[0]["mem_limit_mib"] = 1                                # index 0 only
    c[1]["mem_limit_mib"] = 2                                # no GPU: BAD_PROFILE
    c[2]["mem_limit_mib"] = 5                                # past the selectors: INVALID
    pod_off = np.array([0, 1, 2, 3, 33, 33], np.uint32)      # then 30 one-slice claims on 4 x 7 slices, then an empty pod
    cn, co = _flat([[0, 1, NONE], [1, 1, 0], [2, 0], [0, 1, 1, 5], [1, 0]])
    other = g.copy()
    other["busy"] = 0x7F                                     # every slice taken outside a rank's own range
    splits = [[0, b, 2] for b in range(3)] if world == 2 else [[0, a, b, 2] for a in range(3) for b in range(a, 3)]
    O.set_selectors(attrs, sels)
    try:
        for bounds in splits:
            copies = [diverged(g, off, bounds, r, other) for r in range(world)]
            for flags in (0, Y.F_EXHAUSTIVE):
                for form in ((cn, co), (None, None)):
                    ref = check(g, copies, off, t, c, pod_off, *form, flags, bounds, f"{bounds} f{flags}", attrs, sels)
                    if form[1] is None:
                        continue
                    assert ref[0][2] == Y.WHY_NO_NODE and ref[1][2] == Y.WHY_CLAIM_NONE
                    assert ref[0][3] == ref[0][4] == Y.ST_BAD_PROFILE and ref[1][3] == 1
                    if flags:                                # 28 levels held at most: claim 3 + 28 blocks
                        assert ref[0][8] == Y.ST_SEARCH_LIMIT and ref[1][8] == 31
                        assert ref[3][31] == 3               # node 1 twice and node 0 once, on whichever ranks
    finally:
        O.set_selectors()
