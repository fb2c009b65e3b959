"""CPU suite: the problems that test place pods (spec §13) at its edges, checked without a GPU.

tests/test_gpu_place_pods_edges.py runs these builders on the device against the C oracle, so the oracle is pinned here
first: every builder's problem, at a size the Python restatement can walk, gives the same bytes on
place_oracle.place_pods and place_oracle.place_pods_naive, and each problem reaches the statuses it exists for.

* long candidate lists: 31 to 1,000 entries, the first entry naming a node at positions 0 to 64, runs of strays after a
  failed visit that cross a 32-entry boundary, a pod listing one node 40 times, a list whose only usable entry is last
* exhausted searches across candidates: the 4,095-, 4,096- and 4,097-descent fixtures of test_pod_search_fixtures.py
  as pods, with limit -> POD, limit -> strays, POD -> limit, limit -> placed, and the limit on the last of 41 candidates
* pod shapes and failure records: 32- and 33-claim pods, empty pods, pods without candidates or with strays only,
  claims invalid by §3 and §10, GPU claims of count 0, 2 and 33, every out_off form, arbitrary claim node fields"""
from types import SimpleNamespace

import numpy as np
import pytest

import test_pod_search_fixtures as F
from test_oracle_properties import _dicts
from test_place_pods import _flat, placed_offsets
from test_pod_mode import _tbl

import place_oracle as P

R = F.R
NONE = 0xFFFFFFFF


def strays(n_node):
    """candidates that name no node of an n_node inventory"""
    return (n_node, n_node + 1000, NONE)


def _mig(profiles):
    c = np.zeros(len(profiles), R.CLAIM_DTYPE)
    c["kind"], c["profile"], c["count"] = R.KIND_MIG, profiles, 1
    return c


def problem(name, g, off, t, claims, pod_off, cands, out_off=None, n_out=None):
    """One place-pods call: cands is a list of candidate lists, or None for the dense form.  n_out defaults to what the
    out_off form needs: n_claim without out_off, the packed slot count with it."""
    pod_off = np.asarray(pod_off, np.uint32)
    if n_out is None:
        n_out = len(claims) if out_off is None else int(max([int(o) + int(s) for o, s in
                                                            zip(out_off, _slots(claims, True))], default=0))
    return SimpleNamespace(name=name, gpus=g, node_off=np.asarray(off, np.uint32), table=t, claims=claims,
                           pod_off=pod_off, cands=cands, out_off=out_off, n_out=n_out, n_node=len(off) - 1)


def cand_arrays(pb):
    return (None, None) if pb.cands is None else _flat(pb.cands)


def _slots(claims, have_off):
    c = claims.copy()
    c["node"] = 0
    return R.claim_slots(c, 1, have_off)


# ---- b. long candidate lists ----------------------------------------------------------------------------------------
LENGTHS = (31, 32, 33, 64, 65, 1000)
FIRSTS = (0, 31, 32, 33, 63, 64)


def long_lists(seed=0, longest=1000):
    """One-GPU MIG nodes: the first third full, the rest free; every pod one 7g claim.  Pod lists (strays before the
    first usable entry; a failed visit on a full node, then a run of 33 strays, then the pod's own free node, then a
    random tail) for every length and first position; a pod listing a full node 40 times; lists whose only usable
    entry is the last; strays after failed visits across the 32- and 64-entry boundaries; and ten pods competing for
    ten shared free nodes in shuffled order, so the order of a node's list decides the answer."""
    rng = np.random.default_rng(seed)
    n_full, n_free = 40, 72
    n = n_full + n_free
    g, off = R.make_inventory([1] * n, mig=True)
    g["busy"][:n_full] = 0xFF
    st_ = strays(n)
    free = iter(range(n_full, n))

    def stray(k):
        return st_[k % 3]

    def tail(m):
        return [int(x) if x < n else stray(int(x)) for x in rng.integers(0, n + 3, m)]

    cands = []
    for L in (min(x, longest) for x in LENGTHS):
        for k in FIRSTS:
            if k >= L:
                continue
            for direct in (False, True):
                a = [stray(j) for j in range(L)]
                if direct:                              # the first usable entry is the pod's free node
                    a[k] = next(free)
                    a[k + 1:] = tail(L - k - 1)
                else:                                   # a failed visit, 33 strays, then the free node
                    a[k] = int(rng.integers(0, n_full))
                    f = min(k + 34, L - 1)
                    if f > k:
                        a[f] = next(free)
                        a[f + 1:] = tail(L - f - 1)
                cands.append(a)
    cands.append([5] * 40 + [stray(j) for j in range(5)] + [next(free)])        # 40 entries of one node's list
    cands.append([stray(j) for j in range(longest - 1)] + [next(free)])        # only the last entry is usable
    cands.append([stray(j) for j in range(64)] + [next(free)])
    cands.append([1] + [stray(j) for j in range(35)] + [2] + [stray(j) for j in range(31)] + [3] +
                 [stray(j) for j in range(40)] + [next(free)])                   # stray runs over 32 and 64
    shared = [next(free) for _ in range(10)]
    for i in range(10):
        order = list(rng.permutation(shared))
        a = []
        for x in order:
            a += [int(x)] + [stray(j) for j in range(int(rng.integers(0, 40)))]
        cands.append(a)
    c = _mig([R.GI_7_SLICE] * len(cands))
    return problem(f"long lists {longest}", g, off, R.default_table(), c, np.arange(len(cands) + 1), cands)


# ---- c. exhausted searches across candidates ------------------------------------------------------------------------
def _fx(name):
    return next(f for f in F.budget_fixtures() if f["name"] == name)


def exhausted():
    """Nodes: the fail_4097 / fail_4096 / fail_4095 / ok_4097 / ok_4096 nodes, a full and six empty copies of the
    fail_4097 node's models, one empty copy of ok_4097's.  Pods: the fixtures' pods, with the outcome sequences in
    EXPECT (statuses with DRA_F_EXHAUSTIVE, then without)."""
    L97, F97, L96, L95, LOK97, LOK96, E97, EOK97 = 0, 1, 2, 3, 4, 5, 6, 12
    f97, f96, f95, ok97, ok96 = (_fx(x) for x in ("fail_4097", "fail_4096", "fail_4095", "ok_4097", "ok_4096"))
    full = f97["gpus"].copy()
    full["busy"] = 0xFFFF
    empty = f97["gpus"].copy()
    empty["busy"] = 0
    eok = ok97["gpus"].copy()
    eok["busy"] = 0
    nodes = [f97["gpus"], full, f96["gpus"], f95["gpus"], ok97["gpus"], ok96["gpus"]] + [empty] * 6 + [eok]
    n = len(nodes)
    s = strays(n)
    g = np.concatenate(nodes)
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in nodes])
    g["node"] = np.repeat(np.arange(n), [len(x) for x in nodes])
    p97, p96, p95, pok97, pok96 = (f["pods"][0] for f in (f97, f96, f95, ok97, ok96))
    SL, OK, POD = R.ST_SEARCH_LIMIT, R.ST_OK, R.ST_POD
    rows = [  # name, pod, candidates, (status, node) with DRA_F_EXHAUSTIVE, status without, a candidate out of budget
        ("limit -> POD", p97, [L97, F97], (SL, NONE), POD, L97),
        ("limit -> strays", p97, [L97, *s], (SL, NONE), POD, L97),
        ("POD -> limit", p97, [F97, L97], (SL, NONE), POD, L97),
        ("limit -> placed", p97, [L97, E97], (OK, E97), OK, L97),
        ("limit on the last of 41", p97, [F97] * 20 + [s[k % 3] for k in range(20)] + [L97], (SL, NONE), POD, L97),
        ("limit thrice -> placed", p97, [L97] * 3 + [E97 + 1], (OK, E97 + 1), OK, L97),
        ("limit, 40 strays -> placed", p97, [L97] + [s[k % 3] for k in range(40)] + [E97 + 2], (OK, E97 + 2), OK, L97),
        ("4096 descents -> POD", p96, [L96, F97], (POD, NONE), POD, None),
        ("4095 descents -> POD", p95, [L95, F97], (POD, NONE), POD, None),
        ("POD, 4096 -> ...", p96, [F97, L96, L97], (None, NONE), POD, None),
        ("ok_4097: limit -> placed", pok97, [LOK97, EOK97], (OK, EOK97), OK, LOK97),
        ("placed first", p97, [E97 + 3, L97], (OK, E97 + 3), OK, None),
        ("ok_4096: placed at the budget", pok96, [F97, LOK96], (OK, LOK96), None, None),
    ]
    c = np.concatenate([r[1] for r in rows])
    pod_off = np.zeros(len(rows) + 1, np.uint32)
    pod_off[1:] = np.cumsum([len(r[1]) for r in rows])
    pb = problem("exhausted", g, off, F.fixture_table(), c, pod_off, [list(r[2]) for r in rows])
    pb.expect = [(r[0], r[3], r[4]) for r in rows]
    pb.probe = [r[5] for r in rows]
    return pb


# ---- d. pod shapes and failure records ------------------------------------------------------------------------------
OUT_FORMS = ("none", "packed", "gaps", "spare")
NODE_FIELDS = ("zero", "none", "n_node", "random")


def shapes(seed=0, form="packed", node_field="zero", n_pod=120, sel=True):
    """MIG nodes of 1-2 GPUs, non-MIG nodes of 2-4 GPUs and one of 32.  Pods interleaved at random: 1g-7g and GPU
    claims, 32- and 33-claim pods, empty pods, pods without candidates or with strays only, claims invalid by §3
    (profile 200, kind 7, GPU count 0 or 33) and by §10 (a selector id past the empty table), GPU claims of count 2;
    each with and without a usable candidate.  sel=False: §3 instead of §10 (oracle/naive.py models no selectors)."""
    rng = np.random.default_rng(seed)
    widths = [1, 2] * 5 + [2, 3, 4] * 3 + [32]
    mig = [True] * 10 + [False] * 10
    parts = [R.make_inventory([w], mig=m)[0] for w, m in zip(widths, mig)]
    g = np.concatenate(parts)
    n = len(widths)
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(widths)
    g["node"] = np.repeat(np.arange(n), widths)
    g["busy"][rng.random(len(g)) < 0.3] = 0x0F
    s = strays(n)
    pods, cands = [], []
    kinds = ["mixed"] * 6 + ["c32", "c33", "empty", "gpu2", "bad3", "bad10", "count0", "count33"]
    for p in range(n_pod):
        k = kinds[int(rng.integers(len(kinds)))]
        if k == "c32":
            c = np.zeros(32, R.CLAIM_DTYPE)
            c["kind"], c["count"] = R.KIND_GPU, 1
        elif k == "c33":
            c = _mig([R.GI_1_SLICE] * 33)
        elif k == "empty":
            c = np.zeros(0, R.CLAIM_DTYPE)
        else:
            m = int(rng.integers(1, 5))
            c = _mig(rng.choice([R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE], m))
            if rng.random() < 0.4:
                c = np.concatenate([c, np.zeros(1, R.CLAIM_DTYPE)])
                c[-1]["kind"], c[-1]["count"] = R.KIND_GPU, 1
            j = int(rng.integers(len(c)))
            if k == "gpu2":
                c[j]["kind"], c[j]["profile"], c[j]["count"] = R.KIND_GPU, 0, 2
            elif k == "bad3":
                if rng.random() < 0.5:
                    c[j]["profile"] = 200
                else:
                    c[j]["kind"] = 7
            elif k == "bad10" and sel:
                c[j]["mem_limit_mib"] = 3                      # kinds GPU and MIG name their selector here
            elif k == "bad10":
                c[j]["kind"] = 3
            elif k in ("count0", "count33"):
                c[j]["kind"], c[j]["profile"], c[j]["count"] = R.KIND_GPU, 0, 0 if k == "count0" else 33
        pods.append(c)
        shape = int(rng.integers(4))                           # none / strays only / usable / usable after strays
        if shape == 0:
            cands.append([])
        elif shape == 1:
            cands.append([s[int(x)] for x in rng.integers(0, 3, int(rng.integers(1, 40)))])
        else:
            a = [int(x) for x in rng.integers(0, n, int(rng.integers(1, 9)))]
            if shape == 3:
                a = [s[j % 3] for j in range(int(rng.integers(30, 70)))] + a
            cands.append(a)
    claims = np.concatenate(pods)
    pod_off = np.zeros(n_pod + 1, np.uint32)
    pod_off[1:] = np.cumsum([len(c) for c in pods])
    nrng = np.random.default_rng(seed + 1000)            # (its own stream: the out_off forms do not depend on it)
    if node_field == "none":
        claims["node"] = NONE
    elif node_field == "n_node":
        claims["node"] = n
    elif node_field == "random":
        claims["node"] = nrng.integers(0, 2 ** 32, len(claims), dtype=np.uint64).astype(np.uint32)
    out_off, n_out = out_form(claims, form, rng)
    return problem(f"shapes {seed} {form} {node_field}", g, off, R.default_table(), claims, pod_off, cands, out_off, n_out)


def out_form(claims, form, rng):
    """(out_off, n_out): none (slot i), packed, permuted with gaps, or packed with spare slots at the end"""
    if form == "none":
        return None, len(claims)
    sl = _slots(claims, True).astype(np.int64)
    if form == "gaps":
        out_off = np.zeros(len(claims), np.uint32)
        pos = 0
        for i in rng.permutation(len(claims)):
            pos += int(rng.integers(0, 3))
            out_off[i] = pos
            pos += int(sl[i])
        return out_off, pos + int(rng.integers(0, 3))
    out_off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32) if len(claims) else np.zeros(0, np.uint32)
    return out_off, int(sl.sum()) + (7 if form == "spare" else 0)


# ---- checks ---------------------------------------------------------------------------------------------------------
def oracle_run(pb, exhaustive, start=None):
    cn, co = cand_arrays(pb)
    return P.place_pods(pb.gpus if start is None else start, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co,
                        pb.out_off, pb.n_out, P.F_EXHAUSTIVE if exhaustive else 0)


def check_against_naive(pb, exhaustive):
    out, pod_node, after = oracle_run(pb, exhaustive)
    oo = pb.out_off if pb.out_off is not None else None
    nout, nnode, nafter = P.place_pods_naive(_dicts(pb.gpus), [int(x) for x in pb.node_off], _tbl(pb.table),
                                             _dicts(pb.claims), [int(x) for x in pb.pod_off], pb.cands, exhaustive,
                                             None if oo is None else [int(x) for x in oo])
    got = [tuple(int(v) for v in r) for r in out]
    for i, r in enumerate(nout):                            # slots no claim owns are left to the caller's zeros
        assert got[i] == (r if r is not None else (0, 0, 0, 0, 0)), f"{pb.name}: slot {i}: {got[i]} != {r}"
    assert [int(x) for x in pod_node] == nnode, pb.name
    for a, b in zip(after, nafter):
        assert (int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) == \
               (b["busy"], b["flags"], b["mem_free_mib"], b["share_cnt"]), pb.name
    return out, pod_node, after


def pod_statuses(pb, out, p):
    """the set of statuses in pod p's slots"""
    oo = pb.out_off if pb.out_off is not None else np.arange(len(pb.claims))
    sl = _slots(pb.claims, pb.out_off is not None)
    return {int(out["status"][int(oo[i]) + k]) for i in range(pb.pod_off[p], pb.pod_off[p + 1]) for k in range(sl[i])}


@pytest.mark.parametrize("exhaustive", [False, True])
def test_long_lists_agree_with_naive(exhaustive):
    pb = long_lists(longest=100)
    out, pod_node, _ = check_against_naive(pb, exhaustive)
    n_full = 40
    for p, a in enumerate(pb.cands[:-10]):                  # each pod takes the first free node of its list
        free = [x for x in a if n_full <= x < pb.n_node]
        assert pod_node[p] == (free[0] if free else NONE), p
    assert (pod_node[-10:] != NONE).all()                   # the shared nodes go one to each competing pod
    assert len(set(pod_node[-10:].tolist())) == 10
    pb = problem("long lists dense", pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, None)
    check_against_naive(pb, exhaustive)


def test_long_lists_reach_their_positions():
    pb = long_lists()
    firsts = {next(i for i, x in enumerate(a) if x < pb.n_node) for a in pb.cands if any(x < pb.n_node for x in a)}
    assert set(FIRSTS) <= firsts and 999 in firsts
    assert set(LENGTHS) <= {len(a) for a in pb.cands}


@pytest.mark.parametrize("exhaustive", [False, True])
def test_exhausted_searches(exhaustive):
    pb = exhausted()
    out, pod_node, _ = check_against_naive(pb, exhaustive)
    for p, (name, (st_ex, node_ex), st_plain) in enumerate(pb.expect):
        st = pod_statuses(pb, out, p)
        if exhaustive:
            if st_ex is not None:
                assert st == {st_ex}, f"{name}: {st}"
            assert pod_node[p] == node_ex, name
        else:
            assert R.ST_SEARCH_LIMIT not in st, name
            if st_plain is not None:
                assert st == {st_plain}, f"{name}: {st}"


def test_exhausted_first_candidates_hit_the_budget():
    """each pod whose sequence names a limit runs out of budget on that candidate alone"""
    pb = exhausted()
    assert sum(x is not None for x in pb.probe) >= 7
    for p, node in enumerate(pb.probe):
        if node is None:
            continue
        c0, c1 = int(pb.pod_off[p]), int(pb.pod_off[p + 1])
        one = problem(pb.expect[p][0], pb.gpus, pb.node_off, pb.table, pb.claims[c0:c1], [0, c1 - c0], [[node]])
        out, got, _ = oracle_run(one, True)
        assert set(out["status"]) == {R.ST_SEARCH_LIMIT} and got[0] == NONE, one.name


@pytest.mark.parametrize("form", OUT_FORMS)
def test_shapes_agree_with_naive(form):
    for seed, node_field in enumerate(NODE_FIELDS):
        pb = shapes(seed, form, node_field, n_pod=60, sel=False)
        for exhaustive in (False, True):
            out, pod_node, _ = check_against_naive(pb, exhaustive)
            st = set(out["status"].tolist())
            assert {R.ST_INVALID, R.ST_POD} <= st, pb.name


def test_shapes_cover_their_cases():
    pb = shapes(0, "packed", "zero")
    out, pod_node, _ = oracle_run(pb, True)
    sizes = np.diff(pb.pod_off)
    assert {0, 32, 33} <= set(sizes.tolist())
    assert (sizes == 33).any() and all(pod_statuses(pb, out, p) == {R.ST_INVALID} for p in np.flatnonzero(sizes == 33))
    assert any(len(a) == 0 for a in pb.cands) and any(a and all(x >= pb.n_node for x in a) for a in pb.cands)
    counts = set(pb.claims["count"][pb.claims["kind"] == R.KIND_GPU].tolist())
    assert {0, 2, 33} <= counts
    assert (pb.claims["profile"] == 200).any()
    oo = pb.out_off
    sel = np.flatnonzero((pb.claims["mem_limit_mib"] == 3) & (pb.claims["kind"] != R.KIND_SHARED))
    assert len(sel) and (out["status"][oo[sel]] == R.ST_INVALID).all()         # §10: a selector id past the table
    # pods with a claim invalid by §3 or §10 fail both in the prep (no usable candidate) and after their visits
    bad = (pb.claims["profile"] == 200) | (pb.claims["kind"] > 2) | (pb.claims["mem_limit_mib"] == 3)
    pods = {int(np.searchsorted(pb.pod_off, i, side="right")) - 1 for i in np.flatnonzero(bad)}
    usable = {p for p in pods if sizes[p] <= 32 and any(x < pb.n_node for x in pb.cands[p])}
    assert usable and pods - usable, (pods, usable)
    assert (pod_node != NONE).sum() >= 8 and (out["status"] == R.ST_OK).sum() >= 16


def test_claim_node_fields_are_ignored():
    for form in OUT_FORMS:
        ref = None
        for node_field in NODE_FIELDS:
            pb = shapes(5, form, node_field)
            got = oracle_run(pb, True)
            if ref is not None:
                assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref)), (form, node_field)
            ref = got
