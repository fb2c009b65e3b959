"""CPU suite: spec §16 — pod capacity: how many copies of a pod each candidate node still takes, counted as the pods
Allocate (§12) would place them.

The C oracle (pod_oracle_capacity in tests/pod_oracles.c, on oracle/dra_oracle.c's pod evaluation) and the pure-Python
restatement (capacity_oracle.capacity_naive, on oracle/naive.py's) share no code, so agreement between them pins the
rule; the two consequences §16 states tie it to the pods Allocate and to the exhaustive UnsuitableNodes."""
import importlib
import json
import os
import re

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings

from conftest import GOLDEN
from test_oracle_properties import _dicts
from test_pod_mode import _mig, _tbl

import capacity_oracle as K
import preempt_problems as PB

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _flat(cands):
    off = np.zeros(len(cands) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in cands])
    return np.array([n for x in cands for n in x], dtype=np.uint32), off


def problem(seed, widths=PB.WIDTHS, n_node=6, n_run=40):
    """A §16 problem from a seeded generator: nodes of the given widths (MIG, non-MIG and mixed, two models, now and then
    an UNAVAILABLE GPU) fragmented by pods the oracle's pods Allocate placed on them, preempt_problems' pending pods (0 to
    33 claims, every kind, groups, invalid claims) and candidate lists (duplicates, strays, long lists, or the dense
    form).  Returns (gpus, node_off, table, claims, pod_off, cands)."""
    D = PB._Rng(np.random.default_rng(seed))
    saved, PB.WIDTHS = PB.WIDTHS, tuple(widths)
    try:
        g, off, mig = PB._inventory(D, n_node)
    finally:
        PB.WIDTHS = saved
    t = R.default_table()
    parts, rpo = [], [0]
    for _ in range(n_run):
        n = D.int(0, n_node - 1)
        parts.append(PB._running_claims(D, n, mig[n], True))
        rpo.append(rpo[-1] + len(parts[-1]))
    rc = np.concatenate(parts) if parts else np.zeros(0, R.CLAIM_DTYPE)
    roo, n_out = R.out_offsets(rc, n_node)
    _, g = PB.O.allocate_pods(g, off, t, rc, np.array(rpo, np.uint32), roo, n_out)
    claims, pod_off, _ = PB._pending(D, n_node)
    return g, off, t, claims, pod_off, PB._cands(D, len(pod_off) - 1, n_node)


def run_both(g, off, t, c, pod_off, cands=None, flags=0, max_copies=64):
    cn, co = (None, None) if cands is None else _flat(cands)
    a = K.capacity(g, off, t, c, pod_off, cn, co, max_copies, flags)
    b = K.capacity_naive(_dicts(g), [int(x) for x in off], _tbl(t), _dicts(c), [int(x) for x in pod_off], cands,
                         bool(flags & K.F_EXHAUSTIVE), max_copies)
    for x, y in zip(a, b):
        assert [int(v) for v in x] == list(y)
    return a


def pairs_of(pod_off, cands, n_node):
    """[(pair, pod, node)] in pair order"""
    out = []
    for p in range(len(pod_off) - 1):
        for n in (range(n_node) if cands is None else cands[p]):
            out.append((len(out), p, int(n)))
    return out


def allocate_count(oracle, g, off, t, pod, n, max_copies, flags):
    """OK pods when the pods Allocate is given max_copies copies of `pod`, all naming node n; they must be a prefix"""
    one = pod.copy()
    one["node"] = n
    c = np.concatenate([one] * max_copies)
    pod_off = (np.arange(max_copies + 1) * len(pod)).astype(np.uint32)
    oo, n_out = R.out_offsets(c, len(off) - 1)
    out, _ = oracle.allocate_pods(g, off, t, c, pod_off, oo, n_out, flags)
    end = np.concatenate([oo[1:], [n_out]]).astype(np.int64)
    ok = [all(out["status"][oo[i]: end[i]].tolist() == [0] * int(end[i] - oo[i]) for i in range(q * len(pod), (q + 1) * len(pod)))
          for q in range(max_copies)]
    placed = sum(ok)
    assert ok == [True] * placed + [False] * (max_copies - placed)
    return placed


# ---- the two oracles agree ---------------------------------------------------------------------------------------------
@settings(max_examples=60, deadline=None, suppress_health_check=list(HealthCheck))
@given(PB.problems())
def test_oracle_matches_naive(pb):
    for flags in (0, K.F_EXHAUSTIVE):
        run_both(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.cands, flags, pb.max_victims + 1)


@pytest.mark.parametrize("seed", range(12))
def test_oracle_matches_naive_on_fragmented_nodes(seed):
    g, off, t, c, pod_off, cands = problem(seed, widths=(0, 1, 2, 3, 8) if seed % 2 else PB.WIDTHS)
    seen = set()
    for flags in (0, K.F_EXHAUSTIVE):
        copies, stop, total, nodes = run_both(g, off, t, c, pod_off, cands, flags, (1, 5, 64)[seed % 3])
        seen |= set(stop.tolist())
        k = 0
        for p in range(len(pod_off) - 1):
            n = len(off) - 1 if cands is None else len(cands[p])
            assert int(total[p]) == int(copies[k: k + n].sum()) and int(nodes[p]) == int((copies[k: k + n] > 0).sum())
            k += n
    assert seen <= {K.ST_OK, K.ST_POD, K.ST_SEARCH_LIMIT, K.ST_INVALID}


# ---- consequence 1: Allocate's number ------------------------------------------------------------------------------------
def test_copies_are_what_pods_allocate_places(oracle):
    checked = 0
    for seed in range(8):
        g, off, t, c, pod_off, cands = problem(100 + seed)
        n_node, max_copies = len(off) - 1, (2, 9)[seed % 2]
        cn, co = (None, None) if cands is None else _flat(cands)
        for flags in (0, K.F_EXHAUSTIVE):
            copies, stop, _, _ = K.capacity(g, off, t, c, pod_off, cn, co, max_copies, flags)
            for k, p, n in pairs_of(pod_off, cands, n_node):
                pod = c[pod_off[p]: pod_off[p + 1]]
                if n >= n_node or len(pod) == 0:
                    assert (copies[k], stop[k]) == ((0, K.ST_POD) if n >= n_node else (max_copies, K.ST_OK))
                    continue
                assert copies[k] == allocate_count(oracle, g, off, t, pod, n, max_copies, flags), (seed, k, p, n)
                assert (stop[k] == K.ST_OK) == (copies[k] == max_copies)
                checked += copies[k] > 0
    assert checked > 40


def test_copies_are_what_pods_allocate_places_with_selectors(oracle):
    """Selector ids on MIG claims (one beyond the table: INVALID), in both oracles' selector contexts: two 8-GPU nodes, the
    second with GPUs 0 and 7 full; selector 1 takes GPUs 0..3 of a node, selector 2 GPUs 6 and 7."""
    g, off = R.make_inventory([8, 8], mig=True)
    g["busy"][[8, 15]] = 0xFF
    t = R.default_table()
    attrs = np.zeros(len(g), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(g)) % 8
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 6))])
    c = _mig(R, [R.GI_1_SLICE, R.GI_1_SLICE, R.GI_1_SLICE, R.GI_3_SLICE, R.GI_3_SLICE])
    c["mem_limit_mib"] = [1, 2, 3, 1, 2]
    pod_off = np.array([0, 1, 2, 3, 5], np.uint32)
    K.set_selectors(attrs, sels); oracle.set_selectors(attrs, sels)
    try:
        for flags in (0, K.F_EXHAUSTIVE):
            copies, stop, total, _ = K.capacity(g, off, t, c, pod_off, max_copies=40, flags=flags)
            assert copies.tolist() == [28, 21, 14, 7, 0, 0, 4, 2]
            assert stop.tolist() == [K.ST_POD] * 4 + [K.ST_INVALID] * 2 + [K.ST_POD] * 2 and total.tolist() == [49, 21, 0, 6]
            for k, p, n in pairs_of(pod_off, None, 2):
                assert copies[k] == allocate_count(oracle, g, off, t, c[pod_off[p]: pod_off[p + 1]], n, 40, flags)
    finally:
        K.set_selectors(); oracle.set_selectors()


# ---- consequence 2: at least one copy == the exhaustive UnsuitableNodes bit ------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
def test_one_copy_is_the_exhaustive_unsuitable_bit(oracle, seed):
    g, off, t, c, pod_off, cands = problem(200 + seed)
    n_node = len(off) - 1
    lists = [list(range(n_node))] * (len(pod_off) - 1) if cands is None else cands
    cn, co = _flat(lists)
    copies, _, _, _ = K.capacity(g, off, t, c, pod_off, cn, co, 3, K.F_EXHAUSTIVE)
    bits = oracle.unsuitable(g, off, t, c, pod_off, cn if len(cn) else np.zeros(1, np.uint32), co, flags=oracle.F_EXHAUSTIVE)
    fits = np.unpackbits(bits, bitorder="little")[: len(copies)].astype(bool)
    assert (fits == (copies >= 1)).all()
    if cands is None:                                    # the dense form is the same pairs
        assert K.capacity(g, off, t, c, pod_off, None, None, 3, K.F_EXHAUSTIVE)[0].tolist() == copies.tolist()


def test_first_fit_is_section_12_not_the_claim_walk_of_section_8(oracle):
    """{1g, 3g} on a GPU with slice 4 busy: §8 walks the claims in order and finds the node suitable only for {3g, 1g};
    §12 without backtracking fails {1g, 3g} as a whole, and so does the capacity count; with the flag one copy fits."""
    g, off = R.make_inventory([1], mig=True, busy=1 << 4)
    t = R.default_table()
    pod_off = np.array([0, 2], np.uint32)
    a = _mig(R, [R.GI_1_SLICE, R.GI_3_SLICE])
    assert [x.tolist() for x in run_both(g, off, t, a, pod_off)[:2]] == [[0], [K.ST_POD]]
    assert [x.tolist() for x in run_both(g, off, t, a, pod_off, flags=K.F_EXHAUSTIVE)[:2]] == [[1], [K.ST_POD]]
    # non-MIG claims first (§12 step 2): {1g, GPU} on a node with one MIG and one plain GPU fits whatever the order
    g, off = R.make_inventory([2], mig=True)
    g["flags"][1] = 0
    b = np.concatenate([_mig(R, [R.GI_7_SLICE]), np.zeros(1, R.CLAIM_DTYPE)])
    b[1]["kind"], b[1]["count"] = R.KIND_GPU, 1
    assert run_both(g, off, t, b, pod_off)[0].tolist() == [1]


# ---- known answers -----------------------------------------------------------------------------------------------------
def test_instances_free_on_an_empty_b200():
    """The recorded B200 row (what `nvidia-smi mig -lgip` prints as Instances Free): 7 x 1g, 4 x 1g.45gb, 3 x 2g, 2 x 3g,
    1 x 4g, 1 x 7g per empty GPU; the dense one-claim call is the per-node table."""
    doc = json.load(open(os.path.join(GOLDEN, "b200_gi_profiles.json")))
    t = R.default_table()
    for p, (size, mask) in enumerate(doc["row"]):
        t[15, p] = (size, 0, mask)
    g, off = R.make_inventory([1, 4], model=15)
    profiles = [R.GI_1_SLICE, R.GI_1_SLICE_REV2, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE, R.GI_8_SLICE]
    c = _mig(R, profiles)
    for flags in (0, K.F_EXHAUSTIVE):
        copies, stop, total, nodes = run_both(g, off, t, c, np.arange(len(c) + 1, dtype=np.uint32), flags=flags)
        assert copies.reshape(-1, 2).tolist() == [[7, 28], [4, 16], [3, 12], [2, 8], [1, 4], [1, 4], [0, 0]]
        assert set(stop.tolist()) == {K.ST_POD} and total.tolist() == [35, 20, 15, 10, 5, 5, 0]
        assert nodes.tolist() == [2] * 6 + [0]
    # gpu-test4.yaml:19-44, {1g, 1g, 2g, 3g} on one parent GPU: one copy per empty GPU
    pod = _mig(R, [R.GI_1_SLICE, R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE], groups=[7, 7, 7, 7])
    for flags in (0, K.F_EXHAUSTIVE):
        assert run_both(g, off, t, pod, np.array([0, 4], np.uint32), flags=flags)[0].tolist() == [1, 4]


def test_search_limit_cap_and_time_slicing():
    t = R.default_table()
    g, off = R.make_inventory([1], mig=True)
    # 7 x 1g then a 7g on one empty GPU: infeasible, and the tree of 1g arrangements is far beyond the budget
    pod = _mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])
    pod_off = np.array([0, 8], np.uint32)
    assert [x.tolist() for x in run_both(g, off, t, pod, pod_off, flags=K.F_EXHAUSTIVE)[:2]] == [[0], [K.ST_SEARCH_LIMIT]]
    assert [x.tolist() for x in run_both(g, off, t, pod, pod_off)[:2]] == [[0], [K.ST_POD]]
    # the cap: 7 x 1g fit, asked for at most 7 -> "at least 7"; asked for 8 -> exactly 7
    one = _mig(R, [R.GI_1_SLICE])
    assert [x.tolist() for x in run_both(g, off, t, one, np.array([0, 1], np.uint32), max_copies=7)[:2]] == [[7], [K.ST_OK]]
    assert [x.tolist() for x in run_both(g, off, t, one, np.array([0, 1], np.uint32), max_copies=8)[:2]] == [[7], [K.ST_POD]]
    # a time-slicing share (no memory limit) ends only with the 16-bit share count
    g, off = R.make_inventory([1], mig=False)
    sh = np.zeros(1, R.CLAIM_DTYPE)
    sh["kind"], sh["count"] = R.KIND_SHARED, 1
    copies, stop, total, nodes = K.capacity(g, off, t, sh, np.array([0, 1], np.uint32), max_copies=65535)
    assert (copies.tolist(), stop.tolist(), total.tolist(), nodes.tolist()) == ([65535], [K.ST_OK], [65535], [1])
    g["share_cnt"][0] = 65500
    assert [x.tolist() for x in run_both(g, off, t, sh, np.array([0, 1], np.uint32), max_copies=65535)[:2]] == [[35], [K.ST_POD]]


def test_strays_duplicates_empty_and_oversized_pods():
    g, off = R.make_inventory([1, 2], mig=True)
    t = R.default_table()
    c = _mig(R, [R.GI_3_SLICE] + [R.GI_1_SLICE] * 33)
    pod_off = np.array([0, 1, 1, 34], np.uint32)             # a 3g pod, an empty pod, a pod of 33 claims
    cands = [[1, 5, 1, NONE, 0], [0, 7], [0, 2]]
    copies, stop, total, nodes = run_both(g, off, t, c, pod_off, cands, max_copies=9)
    assert copies.tolist() == [4, 0, 4, 0, 2, 9, 0, 0, 0]
    assert stop.tolist() == [K.ST_POD] * 5 + [K.ST_OK, K.ST_POD, K.ST_INVALID, K.ST_POD]
    assert total.tolist() == [10, 9, 0] and nodes.tolist() == [3, 1, 0]     # a node listed twice is counted twice
    # a pod without candidates, and no pods at all
    assert [x.tolist() for x in run_both(g, off, t, c[:1], np.array([0, 1], np.uint32), [[]])] == [[], [], [0], [0]]
    assert [len(x) for x in K.capacity(g, off, t, None, np.zeros(1, np.uint32))] == [0, 0, 0, 0]


@pytest.mark.parametrize("kw", [dict(flags=1), dict(flags=8), dict(max_copies=0), dict(max_copies=65536),
                                dict(pod_off=[0, 2]), dict(pod_off=[1, 1]), dict(pod_off=[0, 2, 1]),
                                dict(cand_off=[1, 1], cand_nodes=[0]), dict(cand_off=[0, 2, 1], cand_nodes=[0, 0], pod_off=[0, 0, 1])])
def test_call_errors(kw):
    g, off = R.make_inventory([1], mig=True)
    a = dict(pod_off=[0, 1], cand_nodes=None, cand_off=None, max_copies=4, flags=0)
    K.capacity(g, off, R.default_table(), _mig(R, [0]), a["pod_off"], None, None, 4, 0)
    a.update(kw)
    with pytest.raises(ValueError):
        K.capacity(g, off, R.default_table(), _mig(R, [0]), a["pod_off"], a["cand_nodes"], a["cand_off"], a["max_copies"],
                   a["flags"])


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_the_binding_has_the_declared_signature(pkg):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dra_alloc.h")).read(), flags=re.S)
    m = re.search(r"int\s+dra_pod_capacity_batch\s*\(([^)]*)\)\s*;", text)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert params == ["dra_ctx* ctx", "const dra_claim_rec* claims", "uint32_t n_claim", "const uint32_t* pod_off",
                      "uint32_t n_pod", "const uint32_t* cand_nodes", "const uint32_t* cand_off", "uint32_t max_copies",
                      "uint16_t* pair_copies", "uint8_t* pair_stop", "uint64_t* pod_total", "uint32_t* pod_nodes",
                      "uint32_t flags"]
    A = pkg.api
    res, args = A.SYMBOLS["dra_pod_capacity_batch"]
    assert res is A._i32 and args == [A._u32 if p.startswith("uint32_t ") else A._vp for p in params]
    assert hasattr(A.load(), "dra_pod_capacity_batch") and A.KERNELS["pod_capacity"] == 0x8000000
    assert "#define DRA_ABI_VERSION 2" in " ".join(open(os.path.join(ROOT, "include", "dra_alloc.h")).read().split())
