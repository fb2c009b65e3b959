"""CPU suite: the problems of tests/test_gpu_pod_capacity_edges.py, pinned without a device.  On each small one the C
oracle (capacity_oracle.capacity) and the Python restatement (capacity_naive) agree, and each problem reaches what the
GPU tests use it for: 32-claim pods placed many times with backtracks at position 16, SEARCH_LIMIT after copies, every
stop status in the walks, sums past 2^32."""
import importlib

import numpy as np
import pytest

from test_gpu_pod_capacity_edges import (EXH, EMPTY, LIMIT, PALETTE, SUM_LISTS, _pods, deep_problems, structural_problems,
                                         sum_problem, walk_inventory, walk_problem)
from test_oracle_properties import _dicts
from test_pod_mode import _tbl
from test_pod_search_fixtures import resumed, search

import capacity_oracle as K

R = importlib.import_module("k8s-dra-driver_b200").records


def _lists(cn, co):
    return None if co is None else [[int(x) for x in cn[co[p]:co[p + 1]]] for p in range(len(co) - 1)]


def both(g, off, t, c, po, cn=None, co=None, mc=64, fl=0):
    a = K.capacity(g, off, t, c, po, cn, co, mc, fl)
    b = K.capacity_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in po], _lists(cn, co),
                         bool(fl & EXH), mc)
    for x, y in zip(a, b):
        assert [int(v) for v in x] == list(y)
    return a


@pytest.mark.parametrize("width", [8, 16, 32])
def test_walk_problems(width):
    """The walks' pairs, both forms: the oracles agree, and the walks reach every stop status and 65,535 copies"""
    t = R.default_table()
    seen = set()
    for n_walk in (1, 3, 5, 9, 31, 33, 130):
        for form in ("cands", "dense"):
            g, off, c, po, cn, co = walk_problem(width, n_walk, form)
            assert (len(po) - 1) * (len(off) - 1) == n_walk if form == "dense" else int(co[-1]) == n_walk
            assert max(np.diff(off.astype(np.int64))) == width or n_walk < 2
            for fl in (0, EXH):
                copies, stop, _, _ = both(g, off, t, c, po, cn, co, 40, fl)
                seen |= {(int(s), int(x) > 0) for s, x in zip(stop, copies)}
    assert {(K.ST_OK, True), (K.ST_POD, False), (K.ST_INVALID, False), (K.ST_SEARCH_LIMIT, True), (K.ST_POD, True)} <= seen
    g, off, c, po, cn, co = walk_problem(width, 64, "cands")          # the heavy pairs at the GPU tests' max_copies
    copies, stop, _, _ = K.capacity(g, off, t, c, po, cn, co, 65535, 0)
    assert copies.max() == 65535 and stop[0] == K.ST_OK and (stop[copies == 0] != K.ST_OK).all()


def test_palette():
    t = R.default_table()
    g, off = walk_inventory(8)
    c, po = _pods(list(PALETTE))
    copies, stop, _, _ = K.capacity(g, off, t, c, po, None, None, 65535, EXH)
    copies, stop = copies.reshape(7, 6), stop.reshape(7, 6)
    assert copies[0].tolist() == [65535, 0, 535, 0, 0, 0]                  # SHARED: a fresh GPU, 65,000 shares taken
    assert (copies[1] == 65535).all() and (stop[2:4] == K.ST_INVALID).all()
    assert copies[4, 3] == 1 and stop[4, 3] == K.ST_SEARCH_LIMIT          # LIMIT on 3 MIG GPUs


def test_deep_problems_backtrack_at_16_on_copy_after_copy(oracle):
    g, off, t, c, po = deep_problems()
    for fl in (0, EXH):
        copies, stop, _, _ = both(g, off, t, c, po, None, None, 65535, fl)
        if fl:
            assert copies[:3].tolist() == [12, 12, 6] and stop[:2].tolist() == [K.ST_SEARCH_LIMIT, K.ST_POD]
        else:
            assert copies[:2].tolist() == [0, 0] and copies[3] > 0    # first fit places no deep pod, but 32 x 1g
        assert (stop[9:12] == K.ST_INVALID).all()
    # the copies on node 0 in turn: the search of every copy but every fourth resumes at position 16
    deep = c[po[0]:po[1]].copy()
    inv = g[:32].copy()
    inv["node"] = 0
    one = np.array([0, 32], np.uint32)
    backtracks = 0
    for k in range(13):
        placed, n, log = search(inv, t, deep, cap=R.EXH_BUDGET + 8)
        backtracks += 16 in {p for p, _, _ in resumed(log)}
        if k == 12:
            assert placed is None and n > R.EXH_BUDGET
            break
        x = deep.copy()
        x["node"] = 0
        oo, n_out = R.out_offsets(x, 1)
        out, inv = oracle.allocate_pods(inv, one, t, x, np.array([0, 32], np.uint32), oo, n_out, oracle.F_EXHAUSTIVE)
        assert (out["status"] == 0).all()
    assert backtracks >= 10


@pytest.mark.parametrize("width", [8, 16, 32])
def test_structural_problems(width):
    g, off, c, po = structural_problems(width)
    t = R.default_table()
    n_node = len(off) - 1
    seen = set()
    for fl in (0, EXH):
        for mc in (1, 8, 100):
            copies, stop, _, _ = both(g, off, t, c, po, None, None, mc, fl)
            seen |= {(int(s), int(x) > 0) for s, x in zip(stop, copies)}
    assert (K.ST_SEARCH_LIMIT, True) in seen and (K.ST_INVALID, False) in seen
    copies, stop, _, _ = K.capacity(g, off, t, c, po, None, None, 65535, EXH)
    rows = copies.reshape(-1, n_node)
    widths = np.diff(off.astype(np.int64))
    assert widths[0] == 0 and widths[-1] == 0 and widths.max() == width
    gpu_pods = [p for p in range(len(po) - 1) if po[p + 1] - po[p] == 1 and c[po[p]]["kind"] == R.KIND_GPU]
    for i, p in enumerate(gpu_pods[:-2]):                 # a GPU claim as wide as its node: one copy there
        assert rows[p, 1 + i] == 1 and widths[1 + i] == c[po[p]]["count"]
    assert (rows[gpu_pods[-1]] == 0).all() and (stop.reshape(-1, n_node)[gpu_pods[-1]] == K.ST_INVALID).all()  # count 33
    assert rows[gpu_pods[-2]].max() == (1 if width == 32 else 0)                                            # count 32
    shared = [p for p in range(len(po) - 1) if po[p + 1] - po[p] == 1 and c[po[p]]["kind"] == R.KIND_SHARED]
    a = len(gpu_pods) - 1                                 # the plain GPUs with 65,534 and 65,535 shares taken
    assert rows[shared[3], a] == 1 and rows[shared[3], a + 1] == 0        # the time-slicing share: one left, none left
    assert rows[shared[0], a + 3] == 8 + 2 and rows[shared[1], a + 3] == 1 and rows[shared[2], a + 3] == 0   # MPS by memory


def test_sum_problems():
    for n_list in SUM_LISTS:
        c, po, cn, co = sum_problem(n_list, 65538)
        g, off = R.make_inventory([1] * 65538, mig=True)
        _, _, total, nodes = K.capacity(g, off, R.default_table(), c, po, cn, co, 65535, 0)
        assert int(total[0]) == 65535 * n_list > 1 << 32 and int(nodes[0]) == n_list
        assert n_list < 32 * 65537 or n_list // 32 * 65535 > 1 << 32      # one lane's share alone passes 2^32
    assert len(EMPTY) == 0 and len(LIMIT) == 8
