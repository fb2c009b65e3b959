"""CPU suite: the problems of tests/why_edges.py against both statements of each reasons oracle (§17 `why`, §18
`place_why`, §19 `preempt_why` and `preempt_place_why`, each stated twice), the (reason, blocking claim) each fixture was
built for, and the reason matrix the fixtures must reach: every (call, flag, reason) cell of CELLS.  This pins what the
device suite (tests/test_gpu_why_edges.py) expects without a GPU."""
import numpy as np
import pytest

from test_oracle_properties import _dicts
from test_pod_mode import _tbl
from test_preempt import _outs

import place_oracle as PL
import place_why_oracle as PW
import preempt_why_oracle as PY
import why_edges as E
import why_oracle as Y

EXH = Y.F_EXHAUSTIVE
UNS, PLACE, PRE, PREPL = "unsuitable", "place", "preempt", "preempt_place"
_FIRST = {Y.ST_OK, Y.ST_NO_CAPACITY, Y.ST_BAD_PROFILE, Y.ST_MEM_LIMIT, Y.ST_INVALID, Y.WHY_NO_NODE}
_JUDGED = _FIRST | {Y.ST_POD}
# (call, flag) -> the reasons its answers must reach on the fixtures: first-fit §17 answers with Allocate's statuses
# (GROUP, never POD); the judged calls never answer GROUP, and SEARCH_LIMIT only with the flag (without it the search
# does not backtrack)
CELLS = {
    (UNS, 0): _FIRST | {Y.ST_GROUP},
    (UNS, EXH): _JUDGED | {Y.ST_SEARCH_LIMIT},
    (PLACE, 0): _JUDGED, (PLACE, EXH): _JUDGED | {Y.ST_SEARCH_LIMIT},
    (PRE, 0): _JUDGED, (PRE, EXH): _JUDGED | {Y.ST_SEARCH_LIMIT},
    (PREPL, 0): _JUDGED, (PREPL, EXH): _JUDGED | {Y.ST_SEARCH_LIMIT},
}
MODE = {(UNS, 0): "ff", (UNS, EXH): "exh", (PLACE, 0): "place0", (PLACE, EXH): "place1", (PRE, 0): "pre0",
        (PRE, EXH): "pre1", (PREPL, 0): "pre0", (PREPL, EXH): "pre1"}


def answer(pb, call, flags, out_off=True, gpus=None):
    """The oracle's reason outputs (pair_why, pair_claim, pod_why, claim_blocks) of one call on pb, from `gpus` (default
    pb.gpus); placing calls with out_off (the packed slots) or without.  Returns (reasons, extra): extra holds the
    placing call's placements / statuses."""
    g = pb.gpus if gpus is None else gpus
    cn, co = (None, None) if pb.dense else (pb.cand_nodes, pb.cand_off)
    oo, n_out = (pb.out_off, pb.n_out) if out_off else (None, len(pb.claims))
    sel = dict(attrs=pb.attrs, sels=pb.sels)
    if pb.sels is not None:                              # the C oracles of Allocate and of the pod calls alike
        Y.O.set_selectors(pb.attrs, pb.sels)
        PL.set_selectors(pb.attrs, pb.sels)
    try:
        if call == UNS:
            return Y.why(g, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, flags, **sel), ()
        if call == PLACE:
            r = PW.place_why(g, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, oo, n_out, flags, **sel)
            return r[3:], r[:3]
        if call == PRE:
            r = PY.preempt_why(g, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.prio, *pb.run, None, cn, co, flags,
                               **sel)
            return r[1:], r[:1]
        r = PY.preempt_place_why(g, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.prio, *pb.run, None, cn, co, oo,
                                 n_out, flags, **sel)
        return r[6:], r[:6]
    finally:
        if pb.sels is not None:
            Y.O.set_selectors()
            PL.set_selectors()


def naive(pb, call, flags, out_off=True):
    """The second statement of the same call: (pair_why, pair_claim, pod_why, claim_blocks) as lists"""
    args = (_dicts(pb.gpus), [int(x) for x in pb.node_off], _tbl(pb.table), _dicts(pb.claims), [int(x) for x in pb.pod_off])
    oo = [int(x) for x in pb.out_off] if out_off else None
    rc, rpo, rpr, ro = pb.run
    run = (_dicts(rc), [int(x) for x in rpo], [int(x) for x in rpr], _outs(ro))
    prio = [int(x) for x in pb.prio]
    ex = bool(flags & EXH)
    cands = None if pb.dense else pb.cands
    if call == UNS:
        return Y.why_naive(*args, cands, ex)
    if call == PLACE:
        return PW.place_why_naive(*args, cands, ex, oo)[3:]
    if call == PRE:
        return PY.preempt_why_naive(*args, prio, cands, ex, *run)[1:]
    return PY.preempt_place_why_naive(*args, prio, cands, ex, *run, oo)[1:]


def same(a, b, what):
    assert [int(x) for x in a[0]] == list(b[0]), f"{what}: pair_why"
    assert [int(x) for x in a[1]] == list(b[1]), f"{what}: pair_claim"
    assert np.asarray(a[2]).tolist() == [list(r) for r in b[2]], f"{what}: pod_why"
    assert [int(x) for x in a[3]] == list(b[3]), f"{what}: claim_blocks"


CALLS = [(c, f) for c in (UNS, PLACE, PRE, PREPL) for f in (0, EXH)]


@pytest.fixture(scope="module", params=E.WIDTHS)
def fixtures(request):
    pb = E.fixtures(request.param)
    return pb, {cf: answer(pb, *cf)[0] for cf in CALLS}


@pytest.mark.parametrize("call,flags", CALLS)
def test_fixtures_agree_with_the_second_statement(fixtures, call, flags):
    pb, ans = fixtures
    same(ans[(call, flags)], naive(pb, call, flags), f"{pb.name} {call} f{flags}")
    if call in (PLACE, PREPL):                           # the slot mode without out_off
        same(answer(pb, call, flags, out_off=False)[0], naive(pb, call, flags, out_off=False),
             f"{pb.name} {call} f{flags} without out_off")


def test_each_fixture_gives_what_it_was_built_for(fixtures):
    pb, ans = fixtures
    checked = 0
    for (call, flags), (why, claim, _, _) in ans.items():
        mode = MODE[(call, flags)]
        for k, (p, n) in enumerate(pb.pairs()):
            want = pb.pods[p].want.get((mode, n))
            if want is None:
                continue
            r, pos = want
            c = Y.WHY_CLAIM_NONE if pos is None else int(pb.pod_off[p]) + pos
            assert (int(why[k]), int(claim[k])) == (r, c), f"{pb.name} {call} f{flags}: {pb.pods[p].name} on node {n}"
            checked += 1
    assert checked > 300


def test_without_out_off_a_gpu_claim_of_many_is_invalid(fixtures):
    pb, _ = fixtures
    for call in (PLACE, PREPL):
        why, claim, _, _ = answer(pb, call, 0, out_off=False)[0]
        for k, (p, n) in enumerate(pb.pairs()):
            if pb.pods[p].name.startswith("gpu_nocap") and n < pb.n_node:
                pos = pb.pods[p].want[("exh", n)][1]
                assert (int(why[k]), int(claim[k])) == (Y.ST_INVALID, int(pb.pod_off[p]) + pos), pb.pods[p].name


def test_the_reason_matrix_is_reached(fixtures):
    pb, ans = fixtures
    for (call, flags), want in CELLS.items():
        got = set(int(x) for x in ans[(call, flags)][0])
        assert got == want, f"{pb.name} {call} f{flags}: missing {want - got}, unexpected {got - want}"


def test_search_levels(fixtures):
    """The blocking MIG claim of a POD / SEARCH_LIMIT fixture is the d-th MIG claim of its pod, not the d-th claim"""
    pb, ans = fixtures
    why, claim, _, _ = ans[(UNS, EXH)]
    seen = set()
    for k, (p, n) in enumerate(pb.pairs()):
        name = pb.pods[p].name
        if not name.startswith(("pod@", "limit@")) or n != 0:
            continue
        d = int(name.split("@d")[1])
        c = pb.claims[pb.pod_off[p]:pb.pod_off[p + 1]]
        migs = np.flatnonzero(c["kind"] == Y.KIND_MIG)
        assert int(claim[k]) - int(pb.pod_off[p]) == migs[d] != d, name
        seen.add((int(why[k]), d))
    assert seen == {(Y.ST_POD, d) for d in E.POD_LEVELS} | {(Y.ST_SEARCH_LIMIT, d) for d in E.LIMIT_LEVELS}


def test_long_pods():
    """First-fit §17 past 32 claims: the oracle names each blocking claim; the second statement agrees on the pods
    short enough for it"""
    pb = E.long_pods()
    why, claim, pod_why, blocks = Y.why(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.cand_nodes,
                                        pb.cand_off, 0)
    for k, (p, n) in enumerate(pb.pairs()):
        want = pb.pods[p].want.get(("ff", n))
        if n >= pb.n_node:
            assert why[k] == Y.WHY_NO_NODE
        elif want is not None:
            c = Y.WHY_CLAIM_NONE if want[1] is None else int(pb.pod_off[p]) + want[1]
            assert (int(why[k]), int(claim[k])) == (want[0], c), pb.pods[p].name
    short = E.Problem("short", pb.gpus, pb.node_off, pb.table, pb.pods[:3])
    same(answer(short, UNS, 0)[0], naive(short, UNS, 0), "long pods")


@pytest.mark.parametrize("k", [31, 32, 33])
def test_ladder_cycles_the_blocking_claim(k):
    g, off, c, cands = E.ladder(k, 100)
    pb = E.Problem("ladder", g, off, E.R.default_table(), [E.Pod("p", c, {}, cands)])
    for flags in (0, EXH):
        why, claim, pod_why, blocks = Y.why(g, off, pb.table, c, pb.pod_off, pb.cand_nodes, pb.cand_off, flags)
        if flags and k > 32:
            assert set(why.tolist()) == {Y.ST_INVALID}
            continue
        assert set(why.tolist()) == {Y.ST_NO_CAPACITY} and claim.tolist() == cands
        assert pod_why[0, Y.ST_NO_CAPACITY] == 100 and blocks.tolist() == np.bincount(cands, minlength=k).tolist()


@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("flags", [0, EXH])
def test_chains_answer_as_built(mirror, flags):
    """The serial hand-off chains' reasons, stated in closed form for the device suite's chains across more nodes than
    warps, against the oracles on chains of 40 nodes"""
    for build, call in ((E.place_chain, PLACE), (E.pp_chain, PREPL)):
        pb, want = build(40, mirror)
        got = answer(pb, call, flags)[0]
        for name, a, b in zip(("pair_why", "pair_claim", "pod_why", "claim_blocks"), got, want):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), (call, name)


@pytest.mark.parametrize("n_node", [1, 31, 33, 1000])
def test_dense_rows_agree(n_node):
    g, off, c, _ = E.ladder(32, 0, n_node)
    pb = E.flat(f"dense {n_node}", g, off, E.R.default_table(), E.cat([c, c[:5], c]), np.array([0, 32, 37, 69]), None,
                dense=True)
    for call, flags in CALLS:
        if n_node <= 33:
            same(answer(pb, call, flags)[0], naive(pb, call, flags), f"{pb.name} {call} f{flags}")
        assert int(answer(pb, call, flags)[0][2].sum()) == 3 * n_node


def test_a_selector_hiding_the_full_gpu_is_bad_profile():
    """Node 0's SOLE GPU is full: a SOLE claim is NO_CAPACITY there, and BAD_PROFILE when its selector hides that GPU
    (the C oracle's statement only: the second statement has no selectors)"""
    pb = E.selector_problem(8)
    for call, flags in CALLS:
        why, claim, _, _ = answer(pb, call, flags)[0]
        r = [(int(a), int(b) - int(pb.pod_off[p])) for (p, n), a, b in zip(pb.pairs(), why, claim) if n == 0]
        assert r == [(Y.ST_NO_CAPACITY, 8), (Y.ST_BAD_PROFILE, 8), (Y.ST_NO_CAPACITY, 8)], (call, flags)
