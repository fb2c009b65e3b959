"""CPU suite: spec §16 "Sharded form" — why splitting the pairs over the ranks gives the single-inventory answer.

The sharded pod capacity lets the rank whose node range holds a pair's candidate node count that pair on its own copy of
the inventory, answers a candidate naming no node in place, and sums each pod's pairs after the merge.  This model does
exactly that with the CPU oracle: every rank holds a DIVERGED copy (the world's state on its own range, something else
outside it), counts only its own pairs, and the merged result must equal the oracle on the world's state for any
partition of the nodes, empty ranges included."""
import numpy as np
import pytest

from test_pod_capacity import R, _flat, problem
from test_pod_mode import _mig

import capacity_oracle as K
import preempt_problems as PB

NONE = 0xFFFFFFFF


def pristine(seed, n_node, widths=PB.WIDTHS):
    """the inventory problem(seed) starts from, before its running pods fragment it"""
    D = PB._Rng(np.random.default_rng(seed))
    saved, PB.WIDTHS = PB.WIDTHS, tuple(widths)
    try:
        return PB._inventory(D, n_node)[0]
    finally:
        PB.WIDTHS = saved


def bounds_of(rng, n_node, world):
    """a random partition of [0, n_node) into world ranges, empty ones likely"""
    cuts = np.sort(rng.integers(0, n_node + 1, world - 1))
    if world > 2 and rng.integers(0, 2):
        cuts[0] = cuts[1]                                    # force an empty range
    return [0] + [int(c) for c in cuts] + [n_node]


def diverged(state, off, bounds, r, other):
    """rank r's copy: the world's state on its own GPU range, `other` everywhere else"""
    g = other.copy()
    a, b = int(off[bounds[r]]), int(off[bounds[r + 1]])
    g[a:b] = state[a:b]
    return g


def pairs(pod_off, cn, co, n_node):
    """(pod, node) of every pair in pair order"""
    n_pod = len(pod_off) - 1
    if co is None:
        return np.repeat(np.arange(n_pod), n_node), np.tile(np.arange(n_node, dtype=np.int64), n_pod)
    return np.repeat(np.arange(n_pod), np.diff(co.astype(np.int64))), cn.astype(np.int64)


def sharded(copies, off, t, claims, pod_off, cn, co, max_copies, flags, bounds):
    """The sharded call's answer: rank r counts, on copies[r], only the pairs whose node lies in its range (its window, as
    a candidate list of its own); strays get 0 copies and POD; the pods' sums are taken over the merged pairs."""
    n_node, n_pod = len(off) - 1, len(pod_off) - 1
    pod, node = pairs(pod_off, cn, co, n_node)
    n_pair = len(node)
    got_c = np.zeros(n_pair, np.uint16)
    got_s = np.full(n_pair, K.ST_POD, np.uint8)
    owner = np.searchsorted(np.asarray(bounds), node, side="right") - 1
    for r in range(len(bounds) - 1):
        mine = np.flatnonzero((node < n_node) & (owner == r))
        if len(mine) == 0:
            continue
        sub_off = np.zeros(n_pod + 1, np.uint32)
        sub_off[1:] = np.cumsum(np.bincount(pod[mine], minlength=n_pod))
        c, s, _, _ = K.capacity(copies[r], off, t, claims, pod_off, node[mine].astype(np.uint32), sub_off, max_copies, flags)
        got_c[mine], got_s[mine] = c, s
    total = np.zeros(n_pod, np.uint64)
    nodes = np.zeros(n_pod, np.uint32)
    np.add.at(total, pod, got_c.astype(np.uint64))
    np.add.at(nodes, pod, (got_c > 0).astype(np.uint32))
    return got_c, got_s, total, nodes


def check(state, copies, off, t, claims, pod_off, cn, co, max_copies, flags, bounds, what):
    ref = K.capacity(state, off, t, claims, pod_off, cn, co, max_copies, flags)
    got = sharded(copies, off, t, claims, pod_off, cn, co, max_copies, flags, bounds)
    for name, x, y in zip(("pair_copies", "pair_stop", "pod_total", "pod_nodes"), got, ref):
        assert x.tobytes() == y.tobytes(), f"{what}: {name}"
    return ref


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
def test_any_partition_gives_the_single_inventory_answer(world):
    """Random problems (strays, duplicates, empty and INVALID pods, dense and candidate forms), random partitions, each
    rank's copy wrong outside its own range: the merged answer is the oracle's on the world's state."""
    rng = np.random.default_rng(world)
    differs, stops = 0, set()
    for seed in range(6):
        n_node = 6 + seed
        g, off, t, c, pod_off, cands = problem(100 * world + seed, n_node=n_node)
        g0 = pristine(100 * world + seed, n_node)
        full = g.copy()
        full["busy"] = 0xFFFF
        cn, co = (None, None) if cands is None else _flat(cands)
        bounds = bounds_of(rng, n_node, world)
        copies = [diverged(g, off, bounds, r, (g0, full)[r % 2]) for r in range(world)]
        for flags in (0, K.F_EXHAUSTIVE):
            for mc in (1, 7, 64):
                ref = check(g, copies, off, t, c, pod_off, cn, co, mc, flags, bounds, f"w{world} seed {seed} f{flags} mc{mc}")
                stops |= set(ref[1].tolist())
                if world > 1:
                    alone = K.capacity(copies[0], off, t, c, pod_off, cn, co, mc, flags)
                    differs += alone[0].tobytes() != ref[0].tobytes()
    assert {K.ST_OK, K.ST_POD, K.ST_INVALID} <= stops
    assert world == 1 or differs > 0                         # the diverged copies matter: one rank alone is wrong


@pytest.mark.parametrize("world", [2, 3])
def test_search_limit_and_the_copy_cap_across_ranks(world):
    """SEARCH_LIMIT pairs, max_copies 1 and 65535 with a time-slicing SHARED pod, strays and duplicates, over ranges that
    split the nodes every way."""
    t = R.default_table()
    g, off = R.make_inventory([1, 1, 2, 1], mig=True)
    g["flags"][4] = 0                                        # node 3: one plain GPU, most of its shares taken
    g["share_cnt"][4] = 65500
    c = _mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE] + [R.GI_1_SLICE, R.GI_3_SLICE])
    sh = np.zeros(1, R.CLAIM_DTYPE)
    sh["kind"], sh["count"] = R.KIND_SHARED, 1
    claims = np.concatenate([c, sh])
    pod_off = np.array([0, 8, 9, 10, 10, 11], np.uint32)    # 7 x 1g + 7g, 1g, 3g, empty, shared
    cn, co = _flat([[0, 1, 2, NONE], [0, 2, 2, 1, 9], [3, 0], [1, NONE], [3, 0, 3, 7]])
    other = g.copy()
    other["busy"] = 0
    other["share_cnt"] = 0
    splits = [[0, b, 4] for b in range(5)] if world == 2 else [[0, a, b, 4] for a in range(5) for b in range(a, 5)]
    for bounds in splits:
        copies = [diverged(g, off, bounds, r, other) for r in range(world)]
        for flags in (0, K.F_EXHAUSTIVE):
            for mc in (1, 65535):
                for form in ((cn, co), (None, None)):
                    ref = check(g, copies, off, t, claims, pod_off, *form, mc, flags, bounds, f"{bounds} f{flags} mc{mc}")
                    if form[1] is not None and flags and mc == 65535:
                        assert ref[1][0] == K.ST_SEARCH_LIMIT             # 7 x 1g + 7g on node 0: out of budget
                        assert ref[0][13] == ref[0][15] == 35              # the 35 shares left on node 3, listed twice
                        assert ref[1][11] == K.ST_OK and ref[0][11] == 65535   # the empty pod on node 1
