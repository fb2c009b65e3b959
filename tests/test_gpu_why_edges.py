"""GPU suite: the reasons calls (spec §17, §18, §19) at their edges, through the C ABI.

Every call writes into sentinel-filled outputs SLACK elements longer than it may write; every output must be byte for
byte the oracle's (tests/test_why_edges.answer, which the CPU suite checks against the second statement of each oracle),
nothing may be written past an output, a pure call leaves the inventory as it found it, and a placing call leaves the
inventory, out and pod_node exactly as its plain twin (dra_place_pods_batch / dra_preempt_place_batch) does on the same
state.

  1. every reason from every copy of the reasons evaluation, at 8, 16 and 32 lanes per pair (tests/why_edges.py): §17 and
     its sharded form (worlds 2 and 3 on one device), §18 and its sharded form, §19 preemption and preempt and place,
     both flags, both slot modes of the placing calls; first-fit §17 on pods of up to 100,000 claims
  3. the §18 reasons walk where the plain walk was tested: the pair-sort rows of up to 8,193 pairs under the four
     candidate distributions, long candidate lists, exhausted searches, the serial hand-off chains across more nodes
     than warps (both mirrors, §18 and §19 preempt and place), DRA_F_FRESH_INVENTORY on a changed live state, no
     candidates after a sorted Allocate, and preempt and place's choice past one warp
  4. the tallies at scale: 100,000 candidates of one pod blocked by one claim or by 31, 32 or 33 claims in turn (§17 and
     §18 sharded too), ragged lists, dense rows of 1, 31, 33 and 1,000 nodes, and blocking claims past 2^16 and 2^24
  6. one context reused across inventories of 8, 32 and 8 lanes, in both forms, the reasons calls interleaved with the
     plain calls, every output checked

Parts 2 (the pair walks' rounds) and 5 (§17 reasons at the pair cap) are not here."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_place_pods_edges as GE
import test_gpu_shard_place_why as SP
import test_gpu_shard_unsuitable_why as SU
import test_place_pods_edges as PE
import shard_world as S
import why_edges as E
import why_oracle as Y
from test_gpu_pod_call_checks import SENTINEL
from test_why_edges import CELLS, EXH, PLACE, PRE, PREPL, UNS, answer

pytestmark = pytest.mark.gpu
R = E.R
SENT, SLACK = SENTINEL, 16
WHY_NAMES = ("pair_why", "pair_claim", "pod_why", "claim_blocks")


@pytest.fixture(scope="module")
def wctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _buf(n, dt):
    return np.full((max(n, 1) + SLACK) * np.dtype(dt).itemsize, SENT, np.uint8).view(dt)


def _p(x):
    return None if x is None else x.ctypes.data_as(C.c_void_p)


def _load(ctx, pb):
    ctx.set_table(pb.table)
    ctx.set_inventory(pb.gpus, pb.node_off)


def _arrays(pb):
    c = np.ascontiguousarray(pb.claims, dtype=R.CLAIM_DTYPE)
    po = np.ascontiguousarray(pb.pod_off, np.uint32)
    if pb.dense:
        return c, po, None, None, (len(po) - 1) * pb.n_node
    cn, co = np.ascontiguousarray(pb.cand_nodes, np.uint32), np.ascontiguousarray(pb.cand_off, np.uint32)
    return c, po, cn, co, int(pb.cand_off[-1])


def _running(pkg, pb):
    rc, rpo, rpr, ro = pb.run
    keep = [np.ascontiguousarray(rc, R.CLAIM_DTYPE), np.ascontiguousarray(rpo, np.uint32),
            np.ascontiguousarray(rpr, np.int32), np.ascontiguousarray(ro, R.OUT_DTYPE)]
    run = pkg.api.RunningPods(keep[0].ctypes.data, len(rc), keep[1].ctypes.data, len(rpo) - 1, keep[2].ctypes.data, None,
                              keep[3].ctypes.data, len(ro))
    return run, keep


def raw(pkg, ctx, call, pb, flags, out_off=True, want=(True, True), plain=False):
    """One call through the C ABI on sentinel-filled outputs.  call: UNS / PLACE / PRE / PREPL; plain: the placing call's
    twin without reasons.  want: (pair_claim, the tallies).  Returns (rc, placements, reasons): the placing outputs
    (out, pod_node[, pod_status, evicted_by]) and the four reason outputs (None where not asked for), each with its
    slack."""
    c, po, cn, co, n_pair = _arrays(pb)
    n_pod, n_claim = len(po) - 1, len(c)
    oo, n_out = (np.ascontiguousarray(pb.out_off, np.uint32), pb.n_out) if out_off else (None, n_claim)
    why = [_buf(n_pair, np.uint8), _buf(n_pair, np.uint32) if want[0] else None,
           _buf(n_pod * Y.WHY_N, np.uint32) if want[1] else None, _buf(n_claim, np.uint32) if want[1] else None]
    wp = [_p(x) for x in why]
    L, h = ctx._lib, ctx._h
    if call == UNS:
        return L.dra_unsuitable_why_batch(h, _p(c), n_claim, _p(po), n_pod, _p(cn), _p(co), *wp, flags), (), why
    if call == PLACE:
        pl = [_buf(n_out, R.OUT_DTYPE), _buf(n_pod, np.uint32)]
        if plain:
            return L.dra_place_pods_batch(h, _p(c), n_claim, _p(po), n_pod, _p(cn), _p(co), _p(oo), _p(pl[0]), n_out,
                                          _p(pl[1]), flags), pl, None
        return L.dra_place_pods_why_batch(h, _p(c), n_claim, _p(po), n_pod, _p(cn), _p(co), _p(oo), _p(pl[0]), n_out,
                                          _p(pl[1]), *wp, flags), pl, why
    run, keep = _running(pkg, pb)
    pr = np.ascontiguousarray(pb.prio, np.int32)
    st = _buf(n_pair, np.uint8)
    if call == PRE:
        return L.dra_preempt_why_batch(h, _p(c), n_claim, _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(run), _p(st),
                                       *wp, flags), [st], why
    pl = [_buf(n_out, R.OUT_DTYPE), _buf(n_pod, np.uint32), _buf(n_pod, np.uint8), _buf(len(pb.run[1]) - 1, np.uint32)]
    if plain:
        return L.dra_preempt_place_batch(h, _p(c), n_claim, _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(run), _p(oo),
                                         _p(pl[0]), n_out, _p(pl[1]), _p(pl[2]), _p(pl[3]), flags), pl, None
    return L.dra_preempt_place_why_batch(h, _p(c), n_claim, _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(run), _p(oo),
                                         _p(pl[0]), n_out, _p(pl[1]), _p(pl[2]), _p(pl[3]), _p(st), *wp, flags), \
        pl + [st], why


def same(what, name, got, ref):
    """got (with its slack) holds ref, then only sentinel bytes"""
    ref = np.ascontiguousarray(np.asarray(ref).ravel()).astype(got.dtype)
    x = got[:ref.size]
    if x.tobytes() != ref.tobytes():
        bad = np.flatnonzero(x != ref)[:5]
        pytest.fail(f"{what}: {name} differs at {bad}: device {x[bad]} oracle {ref[bad]}")
    assert (got[ref.size:].view(np.uint8) == SENT).all(), f"{what}: written past {name}"


_MEMO = {}


def _oracle(pb, call, flags, out_off, gpus):
    key = (call, flags, out_off, pb.dense, pb.sels is not None, gpus.tobytes(), pb.claims.tobytes(), pb.pod_off.tobytes(),
           pb.cand_nodes.tobytes(), pb.cand_off.tobytes(), pb.prio.tobytes(), *(x.tobytes() for x in pb.run))
    if key not in _MEMO:
        _MEMO.clear() if len(_MEMO) > 64 else None
        _MEMO[key] = answer(pb, call, flags, out_off, gpus=gpus)
    return _MEMO[key]


def check(pkg, ctx, call, pb, flags, what, out_off=True, want=(True, True), ref=None, start=None):
    """One reasons call on the context's live state against the oracle (ref: its reason outputs, when the caller has
    them; else the placements and statuses are checked too; start: the state the call starts from, when not the live
    one), then its plain twin from the same state for a placing call.  Returns the device's pair_why."""
    before = ctx.get_inventory()
    extra = None
    if ref is None:
        ref, extra = _oracle(pb, call, flags, out_off, before if start is None else start)
    rc, pl, why = raw(pkg, ctx, call, pb, flags, out_off, want)
    assert rc == pkg.api.OK, f"{what}: rc {rc} {ctx._lib.dra_last_error(ctx._h)}"
    for name, got, r in zip(WHY_NAMES, why, ref):
        if got is not None:
            same(what, name, got, r)
    after = ctx.get_inventory()
    if extra is not None and call == PRE:
        same(what, "pair_status", pl[0], extra[0])
    elif extra is not None and call == PLACE:
        same(what, "out", pl[0], extra[0]); same(what, "pod_node", pl[1], extra[1])
        assert after.tobytes() == extra[2].tobytes(), f"{what}: inventory differs from the oracle"
    elif extra is not None and call == PREPL:
        for k, name in enumerate(("out", "pod_node", "pod_status", "evicted_by")):
            same(what, name, pl[k], extra[k])
        same(what, "pair_status", pl[4], extra[5])
        assert after.tobytes() == extra[4].tobytes(), f"{what}: inventory differs from the oracle"
    if call in (UNS, PRE):
        assert after.tobytes() == before.tobytes(), f"{what}: a pure call wrote the inventory"
        return why[0]
    ctx.set_inventory(before if start is None else start, pb.node_off)      # (DRA_F_FRESH_INVENTORY: start pristine)
    rc, twin, _ = raw(pkg, ctx, call, pb, flags, out_off, want, plain=True)
    assert rc == pkg.api.OK, what
    for k, (a, b) in enumerate(zip(pl, twin)):
        assert a.tobytes() == b.tobytes(), f"{what}: placing output {k} differs from the call without reasons"
    assert ctx.get_inventory().tobytes() == after.tobytes(), f"{what}: inventory differs from the call without reasons"
    return why[0]


# ---- 1. every reason from every reasons copy, at each lane width ----------------------------------------------------
CALLS = [(c, f) for c in (UNS, PLACE, PRE, PREPL) for f in (0, EXH)]


@pytest.mark.parametrize("width", E.WIDTHS)
def test_every_reason_at_each_lane_width(pkg, wctx, width):
    pb = E.fixtures(width)
    widest = int(np.diff(pb.node_off.astype(np.int64)).max())
    assert width // 2 < widest <= width
    _load(wctx, pb)
    for call, flags in CALLS:
        reasons = set()
        for out_off in ((True, False) if call in (PLACE, PREPL) else (True,)):
            for want in ((True, True), (False, False)):
                wctx.set_inventory(pb.gpus, pb.node_off)
                got = check(pkg, wctx, call, pb, flags, f"w{width} {call} f{flags} off {out_off} want {want}", out_off,
                            want)
                if out_off:
                    reasons |= set(got[:len(pb.pairs())].tolist())
        assert reasons == CELLS[(call, flags)], (width, call, flags)
    wctx.reset_inventory()
    assert wctx.get_inventory().tobytes() == pb.gpus.tobytes(), "the pristine inventory changed"


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("width", E.WIDTHS)
def test_every_reason_sharded(pkg, world, width):
    """The sharded §17 and §18 reasons on the same fixtures: every rank's outputs the oracle's on the world's state"""
    pb = E.fixtures(width)
    cands = (pb.cand_nodes, pb.cand_off)
    bounds = S.bounds(pb.n_node, world, "even")
    W = SU._world(pkg, pb.gpus, pb.node_off, pb.table, world, bounds)
    try:
        for flags in (0, EXH):
            ref = SU._check(W, pb.claims, pb.pod_off, cands, flags, SU.ALL, f"sharded w{width} f{flags}")
            assert set(ref[0].tolist()) == CELLS[(UNS, flags)]
    finally:
        W.close()
    w = pb
    W = SP._world(pkg, w, world, bounds)
    try:
        for flags in (0, EXH):
            ref = SP._check(W, w, pb.claims, pb.pod_off, pb.cand_nodes, pb.cand_off, pb.out_off, pb.n_out, flags,
                            f"sharded place w{width} f{flags}")
            assert set(ref[3].tolist()) == CELLS[(PLACE, flags)]
    finally:
        W.close()


def test_a_selector_hiding_the_full_gpu(pkg, wctx):
    """BAD_PROFILE where a SOLE claim's selector hides the one GPU offering its profile, NO_CAPACITY where it does not"""
    pb = E.selector_problem(8)
    _load(wctx, pb)
    wctx.set_gpu_attrs(pb.attrs); wctx.set_selectors(pb.sels)
    try:
        for call, flags in CALLS:
            wctx.set_inventory(pb.gpus, pb.node_off)
            got = check(pkg, wctx, call, pb, flags, f"selectors {call} f{flags}")
            assert got[2] == Y.ST_BAD_PROFILE and got[0] == Y.ST_NO_CAPACITY
    finally:
        wctx.set_selectors(None); wctx.set_gpu_attrs(None)


def test_first_fit_on_long_pods(pkg, wctx):
    """First-fit §17 on pods of up to 100,000 claims: blocking claims at 32, 255, 256, 65,535 and 99,999, OK exactly
    where dra_unsuitable_batch sets its bit; the sharded form alike"""
    pb = E.long_pods()
    _load(wctx, pb)
    why = check(pkg, wctx, UNS, pb, 0, "long pods")
    n_pair = len(pb.pairs())
    bits = wctx.unsuitable(pb.claims, pb.pod_off, pb.cand_nodes, pb.cand_off, 0)
    ok = np.unpackbits(np.asarray(bits, np.uint8), bitorder="little")[:n_pair].astype(bool)
    assert (ok == (why[:n_pair] == Y.ST_OK)).all() and ok.any()
    W = SU._world(pkg, pb.gpus, pb.node_off, pb.table, 2, [0, 1, 2])
    try:
        SU._check(W, pb.claims, pb.pod_off, (pb.cand_nodes, pb.cand_off), 0, SU.ALL, "long pods sharded")
    finally:
        W.close()


# ---- 3. the §18 reasons walk at the plain walk's edges --------------------------------------------------------------
def _as_problem(pe):
    pb = E.Problem(pe.name, pe.gpus, pe.node_off, pe.table, [E.Pod(str(p), pe.claims[pe.pod_off[p]:pe.pod_off[p + 1]],
                                                                    {}, list(pe.cands[p]))
                                                             for p in range(len(pe.pod_off) - 1)])
    pb.out_off, pb.n_out = None, len(pb.claims)
    return pb


@pytest.mark.parametrize("name", ["long_lists", "exhausted"])
def test_place_walk_edges(pkg, wctx, name):
    """Chosen positions 0, 31, 32, 33, 63 and 64 with runs of dry runs across the 32-entry scans; the sticky limit bit:
    SEARCH_LIMIT with the flag, POD without"""
    pb = _as_problem(PE.long_lists(seed=1) if name == "long_lists" else PE.exhausted())
    for flags in (0, EXH):
        for call in (PLACE, PREPL):
            _load(wctx, pb)
            got = check(pkg, wctx, call, pb, flags, f"{name} {call} f{flags}", out_off=False)
            if name == "exhausted" and call == PLACE:
                assert (Y.ST_SEARCH_LIMIT in got[:len(pb.pairs())]) == bool(flags)


# ---- 4. tallies at scale --------------------------------------------------------------------------------------------
def _expand(small, cands, n_claim, base):
    """the answers of a one-pod problem whose candidates are its nodes once each, for candidates `cands` (each pair on
    the same node gets the same answer: the pod fails everywhere, so no state changes), its claims moved to `base`"""
    why, claim = np.asarray(small[0]), np.asarray(small[1]).astype(np.int64)
    cands = np.asarray(cands)
    w, c = why[cands], claim[cands]
    c = np.where(c == Y.WHY_CLAIM_NONE, Y.WHY_CLAIM_NONE, c + base).astype(np.uint32)
    row = np.bincount(w, minlength=Y.WHY_N).astype(np.uint32)
    blocks = np.bincount(c[c != Y.WHY_CLAIM_NONE].astype(np.int64), minlength=n_claim).astype(np.uint32)
    return w.astype(np.uint8), c, row, blocks


def _tally_problem(k_claims, n_cand, n_node=None):
    g, off, c, cands = E.ladder(k_claims, n_cand, n_node)
    return E.Problem(f"ladder {k_claims} x {n_cand}", g, off, R.default_table(), [E.Pod("p", c, {}, cands)])


@pytest.mark.parametrize("k,n_node", [(1, 1), (32, 32), (33, 33), (31, 31), (32, 1)])
def test_tallies_of_100000_candidates(pkg, wctx, k, n_node):
    """One pod, 100,000 candidates: all blocked by one claim, or by 31, 32, 33 distinct claims in turn (a warp's 32
    pairs name 32 distinct claims, or one repeats)"""
    pb = _tally_problem(k, 100_000, n_node)
    small = _tally_problem(k, pb.n_node, pb.n_node)
    _load(wctx, pb)
    for call, flags in CALLS:
        if k > 32 and call != UNS:
            continue
        s = answer(small, call, flags)[0]
        w, c, row, blocks = _expand(s, pb.cands[0], len(pb.claims), 0)
        check(pkg, wctx, call, pb, flags, f"{pb.name} {call} f{flags}", out_off=False, ref=(w, c, row[None, :], blocks))
    W = SU._world(pkg, pb.gpus, pb.node_off, pb.table, 3, S.bounds(pb.n_node, 3, "uneven"), max_pairs=1 << 17)
    try:
        for flags in (0, EXH):
            w, c, row, blocks = _expand(answer(small, UNS, flags)[0], pb.cands[0], len(pb.claims), 0)
            for r, got in enumerate(SU._why(W, pb.claims, pb.pod_off, (pb.cand_nodes, pb.cand_off), flags)):
                S.same(got, (w, c, row[None, :], blocks), WHY_NAMES, f"{pb.name} sharded f{flags} rank {r}")
    finally:
        W.close()
    if k > 32:
        return
    W = SP._world(pkg, pb, 3, S.bounds(pb.n_node, 3, "uneven"), max_pairs=1 << 17)
    try:
        for flags in (0, EXH):
            w, c, row, blocks = _expand(answer(small, PLACE, flags, out_off=False)[0], pb.cands[0], len(pb.claims), 0)
            plain = S.place(W, pb.claims, pb.pod_off, (pb.cand_nodes, pb.cand_off), None, len(pb.claims), flags)
            res = SP._why(W, pb.claims, pb.pod_off, (pb.cand_nodes, pb.cand_off), None, len(pb.claims), flags)
            for r, (table, got) in enumerate(res):
                assert table.tobytes() == plain[r][0].tobytes(), f"{pb.name} sharded place f{flags} rank {r}"
                S.same(got, (plain[r][1], w, c, row[None, :], blocks), SP.NAMES, f"{pb.name} sharded place rank {r}")
    finally:
        W.close()


@pytest.mark.parametrize("n_cand", [1, 31, 32, 33])
def test_ragged_lists(pkg, wctx, n_cand):
    pb = _tally_problem(32, n_cand, 32)
    _load(wctx, pb)
    for call, flags in CALLS:
        check(pkg, wctx, call, pb, flags, f"{pb.name} {call} f{flags}", out_off=False)


def test_blocking_claims_past_2_16_and_2_24(pkg, wctx):
    """A claims array of 2^24 + 64 claims: pods without candidates up to 2^16 and 2^24, ladder pods of 32 claims at
    2^16, 2^24 and 2^24 + 32, each with 1,000 candidates; claim_blocks past 2^24 exact, and with pair_claim NULL"""
    g, off, lad, cands = E.ladder(32, 1000)
    n_claim = (1 << 24) + 64
    claims = np.zeros(n_claim, R.CLAIM_DTYPE)
    claims["kind"] = R.KIND_SHARED
    bases = [1 << 16, 1 << 24, (1 << 24) + 32]
    for b in bases:
        claims[b:b + 32] = lad
    pod_off = np.array([0, 1 << 16, (1 << 16) + 32, 1 << 24, (1 << 24) + 32, n_claim], np.uint32)
    pb = E.Problem("2^24 claims", g, off, R.default_table(), [E.Pod("p", lad, {}, cands)])
    pb.claims, pb.pod_off = claims, pod_off
    pb.cands = [[], cands, [], cands, cands]
    pb.cand_off = np.array([0, 0, 1000, 1000, 2000, 3000], np.uint32)
    pb.cand_nodes = np.array(cands * 3, np.uint32)
    pb.prio = np.full(5, E.PRIO, np.int32)
    pb.out_off, pb.n_out = None, n_claim
    small = _tally_problem(32, 32)
    _load(wctx, pb)
    for call, flags in ((UNS, 0), (UNS, EXH), (PLACE, 0), (PRE, EXH)):
        s = answer(small, call, flags)[0]
        parts = [_expand(s, cands, n_claim, b) for b in bases]
        row = np.zeros((5, Y.WHY_N), np.uint32)
        row[[1, 3, 4]] = [p[2] for p in parts]
        ref = (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), row,
               sum(p[3] for p in parts))
        assert ref[3][(1 << 24) + 40] == sum(1 for n in cands if n == 8)
        for want in ((True, True), (False, True)):
            check(pkg, wctx, call, pb, flags, f"2^24 {call} f{flags} want {want}", out_off=False, want=want, ref=ref)


# ---- 6. one context reused ------------------------------------------------------------------------------------------
def test_context_reused_across_widths(pkg, oracle, wctx):
    """Inventories of 8, 32 and 8 lanes on one context, the reasons calls growing and shrinking in pods, pairs and
    claims, in both forms, each optional output on and off, with place pods, preemption, capacity and Allocate between
    them, every output checked"""
    import capacity_oracle as K
    import place_oracle as PO
    import preempt_oracle as PR
    for i, width in enumerate((8, 32, 8)):
        pb = E.fixtures(width)
        _load(wctx, pb)
        cut = E.Problem(f"w{width} cut", pb.gpus, pb.node_off, pb.table, pb.pods[i::2], pb.run)
        dense = E.Problem(f"w{width} dense", pb.gpus, pb.node_off, pb.table, pb.pods[i::5], pb.run, dense=True)
        for j, sub in enumerate((pb, cut, dense, pb) if i != 1 else (cut, dense, pb, cut)):
            for call, flags in CALLS[j % 2::2]:
                want = ((j + i) % 2 == 0, (j + i) % 3 != 0)
                check(pkg, wctx, call, sub, flags, f"reuse {i}.{j} {sub.name} {call} f{flags}", want=want)
            # the plain calls sharing the staging, each against its oracle
            what = f"reuse {i}.{j} {sub.name}"
            cn, co = (None, None) if sub.dense else (sub.cand_nodes, sub.cand_off)
            before = wctx.get_inventory()
            bits = wctx.unsuitable(sub.claims, sub.pod_off, cn, co, 0)
            assert bits.tobytes() == oracle.unsuitable(before, sub.node_off, sub.table, sub.claims, sub.pod_off,
                                                       sub.cand_nodes, sub.cand_off).tobytes(), what
            got = wctx.preempt(sub.claims, sub.pod_off, sub.prio, *sub.run, cand_nodes=cn, cand_off=co, max_victims=4)
            ref = PR.preempt(before, sub.node_off, sub.table, sub.claims, sub.pod_off, sub.prio, *sub.run, None, cn, co,
                             max_victims=4)
            for a, b in zip(got, ref):
                assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), f"{what} preempt"
            got = wctx.pod_capacity(sub.claims, sub.pod_off, cn, co, 8, exhaustive=bool(j % 2))
            ref = K.capacity(before, sub.node_off, sub.table, sub.claims, sub.pod_off, cn, co, 8,
                             K.F_EXHAUSTIVE if j % 2 else 0)
            for a, b in zip(got, ref):
                assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), f"{what} capacity"
            got = wctx.place_pods(sub.claims, sub.pod_off, cn, co, sub.out_off, sub.n_out)
            ref = PO.place_pods(before, sub.node_off, sub.table, sub.claims, sub.pod_off, cn, co, sub.out_off, sub.n_out)
            assert got[0].tobytes() == ref[0].tobytes() and got[1].tobytes() == ref[1].tobytes(), f"{what} place"
            assert wctx.get_inventory().tobytes() == ref[2].tobytes(), f"{what} place inventory"
            # an Allocate of the pods' claims on node 0, then back to the fixtures' inventory
            c = sub.claims.copy()
            c["node"] = 0
            oo, n_out = R.out_offsets(c, sub.n_node)
            live = wctx.get_inventory()
            out = wctx.allocate(c, oo, n_out)
            ref_out, ref_inv = oracle.allocate(live, sub.node_off, sub.table, c, oo, n_out)
            assert out.tobytes() == ref_out.tobytes() and wctx.get_inventory().tobytes() == ref_inv.tobytes(), what
            wctx.set_inventory(pb.gpus, pb.node_off)


# ---- 3 (cont.). the §18 reasons walk on the plain walk's other edges --------------------------------------------------
SMALL_ROWS = [r for r in GE.ROWS if r[1](132)[0] <= 8_193]


@pytest.mark.parametrize("row,dist", [pytest.param(r, d, id=f"{r[0]}-{d}") for r in SMALL_ROWS for d in GE.D4])
def test_pair_sort_rows(pkg, wctx, row, dist):
    """The pair-sort rows of up to 8,193 pairs (the one-CTA sort at its pair and shared-memory limits, the first
    CTA-wide histogram): every reasons output the oracle's, the placements the plain call's, the
    sort chain and histogram tile the plain call's"""
    name, shape, chain, tile, both = row
    n_pair, n_node = shape(GE._n_sm())
    pe, cn, co = GE.sort_workload(R, n_pair, n_node, dist)
    cands = [cn[co[p]:co[p + 1]].tolist() for p in range(len(co) - 1)]
    pb = E.flat(pe.name, pe.gpus, pe.node_off, pe.table, pe.claims, pe.pod_off, cands)
    for flags in ((0, EXH) if both else (0,)):
        _load(wctx, pb)
        check(pkg, wctx, PLACE, pb, flags, f"{name} {dist} f{flags}", out_off=False)
        _load(wctx, pb)
        assert raw(pkg, wctx, PLACE, pb, flags, out_off=False)[0] == pkg.api.OK
        got = wctx.last_chain()
        assert chain - {"place"} <= got, f"{name}: took {sorted(got)}"
        assert wctx.last_hist_tile() == tile, f"{name}: hist tile {wctx.last_hist_tile()}"


@pytest.mark.parametrize("mirror", [False, True])
def test_serial_chains(pkg, wctx, mirror):
    """The hand-off chains across more nodes than warps, §18 and §19 preempt and place: the closed-form reasons
    (tests/test_why_edges.py checks them against the oracles on short chains)"""
    n = GE._n_wide()
    for build, call in ((E.place_chain, PLACE), (E.pp_chain, PREPL)):
        pb, ref = build(n, mirror)
        for flags in (0, EXH):
            _load(wctx, pb)
            check(pkg, wctx, call, pb, flags, f"{pb.name} {call} f{flags}", out_off=False, ref=ref)


def test_fresh_inventory_on_a_changed_live_state(pkg, wctx):
    """A first place pods call puts a 1g on every node; reasons calls with DRA_F_FRESH_INVENTORY then start from the
    pristine state, in both forms"""
    A = pkg.api
    n = GE._n_wide()
    rng = np.random.default_rng(9)
    g, off = R.make_inventory([2] * n, mig=True)
    t = R.default_table()
    first = E.flat("1g everywhere", g, off, t, E.cat([E.mig(R.GI_1_SLICE)] * n), np.arange(n + 1), [[i] for i in range(n)])
    c = E.cat([E.mig(int(x)) for x in rng.choice([R.GI_3_SLICE, R.GI_4_SLICE, R.GI_7_SLICE], 120)])
    pb = E.flat("fresh", g, off, t, c, np.arange(121), [[int(x) for x in rng.integers(0, n + 2, 8)] for _ in range(120)])
    few = E.flat("fresh dense", g, off, t, c[:1], np.arange(2), None, dense=True)
    _load(wctx, first)
    for flags in (A.F_FRESH_INVENTORY, A.F_FRESH_INVENTORY | EXH):
        for sub in (pb, few):
            wctx.place_pods(first.claims, first.pod_off, first.cand_nodes, first.cand_off)
            assert (wctx.get_inventory()["busy"] != g["busy"]).any()
            check(pkg, wctx, PLACE, sub, flags, f"{sub.name} f{flags}", out_off=False, start=g)


def test_no_candidates_after_a_sorted_allocate(pkg, oracle):
    """The candidate form with no candidate at all, after an Allocate on the sorting chain: no pair record written, and
    zero tally rows, for §18 and §19 preempt and place"""
    A = pkg.api
    w = pkg.synth.mixed(600, 8, 5)
    with A.Context(device=0, flags=A.CFG_NO_FUSED) as ctx:
        ctx.set_table(w.table)
        ctx.set_inventory(w.gpus, w.node_off)
        for call in (PLACE, PREPL):
            for flags in (0, EXH):
                out = ctx.allocate(w.claims, w.out_off, w.n_out)
                assert not {"fused_staged", "fused_stream", "fused_direct"} & ctx.last_chain()
                pb = E.flat("no candidates", w.gpus, w.node_off, w.table, w.claims[:6].copy(),
                            np.array([0, 2, 4, 6], np.uint32), [[], [], []])
                live = ctx.get_inventory()
                ref, inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
                assert out.tobytes() == ref.tobytes() and live.tobytes() == inv.tobytes()
                check(pkg, ctx, call, pb, flags, f"no candidates {call} f{flags}")
                ctx.set_inventory(w.gpus, w.node_off)


def test_choice_past_one_warp(pkg, wctx):
    """Preempt and place with 70 candidates per pod: pod 0's best node at positions 5, 6, 37 and 69"""
    from test_gpu_preempt_edges import _warp_world
    g, off, rc, rpo, rpr, ro = _warp_world(R)
    stray = [3, 4, E.NONE]
    a = [stray[k % 3] if k % 4 else 1 for k in range(70)]
    for k in (0, 2, 33, 36, 64):
        a[k] = 2
    for k in (5, 6, 37, 69):
        a[k] = 0
    b = [2 if k % 3 == 0 else 1 if k % 3 == 1 else stray[k % 2] for k in range(70)]
    b[63], b[64] = 0, 0
    pb = E.flat("past one warp", g, off, R.default_table(), E.cat([E.mig(R.GI_7_SLICE)] * 2), np.array([0, 1, 2]),
                [a, b], (rc, rpo, rpr, ro), prio=100)
    for flags in (0, EXH):
        for out_off in (True, False):
            _load(wctx, pb)
            check(pkg, wctx, PREPL, pb, flags, f"past one warp f{flags} off {out_off}", out_off=out_off)


@pytest.mark.parametrize("n_node", [1, 31, 33, 1000])
def test_dense_rows(pkg, wctx, n_node):
    """Dense rows: three pods against every node of a ladder of n_node nodes"""
    g, off, c, _ = E.ladder(32, 0, n_node)
    pb = E.flat(f"dense {n_node}", g, off, R.default_table(), E.cat([c, c[:5], c]), np.array([0, 32, 37, 69]), None,
                dense=True)
    for call, flags in CALLS:
        _load(wctx, pb)
        check(pkg, wctx, call, pb, flags, f"{pb.name} {call} f{flags}")
