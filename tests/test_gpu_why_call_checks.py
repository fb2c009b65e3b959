"""GPU suite: what the six reasons calls (spec §17–§19) promise about their arguments, their outputs and their world.
The four synchronous calls (UnsuitableNodes, place pods, preemption, preempt and place, each with reasons) and the two
sharded ones (UnsuitableNodes and place pods, at world 1 and 2 on one device) are called through the raw ABI into
sentinel-filled outputs with slack past the end:
- a refused call returns its code, writes no output byte and no live or pristine inventory word, and launches nothing;
- where two arguments are wrong, the code says which check comes first;
- a valid call, with pair_why alone, with each optional output added alone and with all four, launches the kernels it is
  known for, reports its chain, and writes exactly the oracle's answer into what was asked for and nothing else;
- a call with claim_blocks after another on the same context counts only its own pairs;
- empty calls launch what they are known for, and a profiled call times the stages its plain twin times."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_pod_call_checks import _world as _pod_world

import place_why_oracle as PW
import preempt_why_oracle as PY
import shard_world as S
import why_oracle as Y

pytestmark = pytest.mark.gpu
SENTINEL = 0xC3
SLACK = 16                                                 # elements past the end of every output
UNS, PLACE, PRE, PREPL = "unsuitable_why", "place_pods_why", "preempt_why", "preempt_place_why"
SYNC = (UNS, PLACE, PRE, PREPL)
SU, SP = "unsuitable_why_shard", "place_pods_why_shard"
CN, CO = [0, 1, 1], [0, 2, 3]                               # a valid candidate form for the two pending pods
NAMES = ("pair_why", "pair_claim", "pod_why", "claim_blocks")
ASKED = [(True, False, False, False), (True, True, False, False), (True, False, True, False), (True, False, False, True),
         (True, True, True, True)]


def _world(R):
    """The two-node world of the pod-call checks, with pod 0 asking for a whole GPU (blocked by the running 1g pod on
    either node: a reason and a blocking claim) and pod 1 for a 1g instance (fits)."""
    w = _pod_world(R)
    w.c["profile"] = [R.GI_7_SLICE, R.GI_1_SLICE]
    return w


@pytest.fixture(scope="module")
def ctx(pkg):
    c = pkg.api.Context(device=0)
    yield c
    c.close()


def _load(ctx, w):
    ctx.set_table(w.t)
    ctx.set_inventory(w.g, w.off)


def _base(w):
    return dict(c=w.c, po=w.po, prio=w.prio, cn=None, co=None, n_out=len(w.c), fl=0, asked=ASKED[-1], null_why=False)


def _n_pair(a, n_node):
    return (len(a["po"]) - 1) * n_node if a["co"] is None else int(a["co"][-1])


def _filled(n, dt):
    return np.full((n + SLACK) * np.dtype(dt).itemsize, SENTINEL, np.uint8).view(dt)


def _raw(pkg, ctx, w, fn, a):
    """dra_<fn> through ctypes on sentinel-filled host outputs; returns (rc, the call's own outputs, the four reasons)"""
    A = pkg.api
    arr = lambda k, dt: None if a.get(k) is None else np.ascontiguousarray(a[k], dtype=dt)   # noqa: E731
    c, po, prio = arr("c", A.R.CLAIM_DTYPE), arr("po", np.uint32), arr("prio", np.int32)
    cn, co = arr("cn", np.uint32), arr("co", np.uint32)
    if cn is not None and not len(cn):
        cn = np.zeros(1, np.uint32)                        # (NULL would mean the dense form)
    n_pod, n_claim, n_out, fl = len(po) - 1, len(c), a["n_out"], a["fl"]
    n_pair = _n_pair(a, ctx.n_node)
    why = [_filled(n_pair, np.uint8), _filled(n_pair, np.uint32), _filled(n_pod * A.WHY_N, np.uint32),
           _filled(n_claim, np.uint32)]
    own = {UNS: [], PLACE: [_filled(n_out, A.R.OUT_DTYPE), _filled(n_pod, np.uint32)], PRE: [_filled(n_pair, np.uint8)],
           PREPL: [_filled(n_out, A.R.OUT_DTYPE), _filled(n_pod, np.uint32), _filled(n_pod, np.uint8),
                   _filled(len(w.rpo) - 1, np.uint32), _filled(n_pair, np.uint8)]}[fn]
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)          # noqa: E731
    wp = [None if (not k or (i == 0 and a["null_why"])) else p(x) for i, (x, k) in enumerate(zip(why, a["asked"]))]
    run = A.RunningPods(w.rc.ctypes.data, len(w.rc), w.rpo.ctypes.data, len(w.rpo) - 1, w.rpr.ctypes.data, None,
                        w.ro.ctypes.data, len(w.ro))
    L, h = ctx._lib, ctx._h
    if fn == UNS:
        rc = L.dra_unsuitable_why_batch(h, p(c), n_claim, p(po), n_pod, p(cn), p(co), *wp, fl)
    elif fn == PLACE:
        rc = L.dra_place_pods_why_batch(h, p(c), n_claim, p(po), n_pod, p(cn), p(co), None, p(own[0]), n_out, p(own[1]), *wp, fl)
    elif fn == PRE:
        rc = L.dra_preempt_why_batch(h, p(c), n_claim, p(po), p(prio), n_pod, p(cn), p(co), C.byref(run), p(own[0]), *wp, fl)
    else:
        rc = L.dra_preempt_place_why_batch(h, p(c), n_claim, p(po), p(prio), n_pod, p(cn), p(co), C.byref(run), None,
                                           p(own[0]), n_out, *[p(x) for x in own[1:]], *wp, fl)
    return rc, own, why


def _oracle(w, g, fn, a):
    """(the call's own outputs, the four reasons, the inventory after) by the oracles, from the inventory g"""
    c, po, cn, co = a["c"], np.asarray(a["po"], np.uint32), a["cn"], a["co"]
    cn = None if cn is None else np.asarray(cn, np.uint32)
    co = None if co is None else np.asarray(co, np.uint32)
    if fn == UNS:
        return [], list(Y.why(g, w.off, w.t, c, po, cn, co, a["fl"])), g
    if fn == PLACE:
        r = PW.place_why(g, w.off, w.t, c, po, cn, co, None, a["n_out"], a["fl"])
        return [r[0], r[1]], list(r[3:]), r[2]
    prio = np.asarray(a["prio"], np.int32)
    if fn == PRE:
        r = PY.preempt_why(g, w.off, w.t, c, po, prio, w.rc, w.rpo, w.rpr, w.ro, None, cn, co, a["fl"])
        return [r[0]], list(r[1:]), g
    r = PY.preempt_place_why(g, w.off, w.t, c, po, prio, w.rc, w.rpo, w.rpr, w.ro, None, cn, co, None, a["n_out"], a["fl"])
    return [r[0], r[1], r[2], r[3], r[5]], list(r[6:]), r[4]


def _same(got, ref, n, what):
    """got (a sentinel-filled output) holds ref in its first n elements and nothing past them"""
    x = got[:n]
    assert x.tobytes() == np.ascontiguousarray(ref, x.dtype).ravel()[:n].tobytes(), f"{what}: {x} != {np.ravel(ref)}"
    assert (got[n:].view(np.uint8) == SENTINEL).all(), f"{what}: written past the end"


def _untouched(outs):
    return all((o.view(np.uint8) == SENTINEL).all() for o in outs)


def _refused(pkg, ctx, w, fn, code, what, **kw):
    n0 = ctx.launch_count()
    rc, own, why = _raw(pkg, ctx, w, fn, dict(_base(w), **kw))
    assert rc == code, f"{fn} {what}: {rc} (expected {code})"
    assert ctx.launch_count() == n0, f"{fn} {what}: launched"
    assert _untouched(own + why), f"{fn} {what}: an output was written"
    assert ctx.get_inventory().tobytes() == w.g.tobytes(), f"{fn} {what}: live inventory changed"
    ctx.reset_inventory()
    assert ctx.get_inventory().tobytes() == w.g.tobytes(), f"{fn} {what}: pristine inventory changed"


CASES = [
    ("unknown flag", SYNC, dict(fl=0x1)),                  # DRA_F_NODE_SORTED: no reasons call takes it
    ("FRESH where not taken", (UNS, PRE, PREPL), dict(fl=0x2)),
    ("pod_off[0] != 0", SYNC, dict(po=[1, 1, 2])),
    ("pod_off[n_pod] != n_claim", SYNC, dict(po=[0, 1, 1])),
    ("cand_nodes without cand_off", SYNC, dict(cn=[0])),
    ("cand_off listing candidates, cand_nodes NULL", SYNC, dict(co=[0, 1, 2])),
    ("cand_off decreasing", SYNC, dict(cn=[0, 1], co=[0, 2, 1])),
    ("pair_why NULL with pairs", SYNC, dict(null_why=True)),
    ("pair_why NULL with candidate pairs", SYNC, dict(null_why=True, cn=CN, co=CO)),
    ("n_out < n_claim", (PLACE, PREPL), dict(n_out=1)),
    ("two faults: unknown flag, pair_why NULL", SYNC, dict(fl=0x1, null_why=True)),
    ("two faults: cand_off decreasing, pair_why NULL", SYNC, dict(cn=[0, 1], co=[0, 2, 1], null_why=True)),
]


@pytest.mark.parametrize("fn", SYNC)
def test_refused_calls_write_nothing(pkg, ctx, oracle, fn):
    A = pkg.api
    w = _world(pkg.records)
    for name, fns, kw in CASES:
        if fn in fns:
            _load(ctx, w)
            _refused(pkg, ctx, w, fn, A.E_INVAL, name, **kw)


@pytest.mark.parametrize("fn", SYNC)
def test_no_inventory_is_checked_after_the_flags_and_before_the_outputs(pkg, fn):
    A = pkg.api
    w = _world(pkg.records)
    with A.Context(device=0) as c:
        c.set_table(w.t)
        for kw, code in ((dict(fl=0x1), A.E_INVAL), (dict(null_why=True), A.E_STATE), ({}, A.E_STATE)):
            n0 = c.launch_count()
            rc, own, why = _raw(pkg, c, w, fn, dict(_base(w), **kw))
            assert rc == code, kw
            assert c.launch_count() == n0 and _untouched(own + why), kw


# (call, form, launches with pair_why alone, chain); a call asked for pod_why or claim_blocks launches k_why_tally too
VALID = [
    (UNS, "dense", 1, {"unsuitable_why"}), (UNS, "cands", 1, {"unsuitable_why"}),
    (PLACE, "dense", 2, {"place", "place_why"}), (PLACE, "cands", 3, {"place", "place_why", "bucket_small"}),
    (PRE, "dense", 4, {"preempt", "unsuitable_why", "bucket_small"}),
    (PRE, "cands", 4, {"preempt", "unsuitable_why", "bucket_small"}),
    (PREPL, "dense", 6, {"preempt_place", "place_why", "bucket_small"}),
    (PREPL, "cands", 7, {"preempt_place", "place_why", "bucket_small"}),
]


def _valid(pkg, ctx, w, fn, a, launches, chain, what):
    _load(ctx, w)
    n0 = ctx.launch_count()
    rc, own, why = _raw(pkg, ctx, w, fn, a)
    assert rc == pkg.api.OK, f"{what}: {ctx._lib.dra_last_error(ctx._h)}"
    tally = a["asked"][2] or a["asked"][3]
    assert ctx.launch_count() - n0 == launches + tally, what
    assert ctx.last_chain() == chain, what
    ref_own, ref_why, ref_inv = _oracle(w, w.g, fn, a)
    for i, (x, y) in enumerate(zip(own, ref_own)):
        _same(x, y, np.asarray(y).size, f"{what}: output {i}")
    for name, x, y, k in zip(NAMES, why, ref_why, a["asked"]):
        if k:
            _same(x, y, np.asarray(y).size, f"{what}: {name}")
        else:
            assert _untouched([x]), f"{what}: {name} written without being asked"
    assert ctx.get_inventory().tobytes() == ref_inv.tobytes(), f"{what}: inventory"


@pytest.mark.parametrize("fn,form,launches,chain", VALID)
def test_valid_calls(pkg, ctx, oracle, fn, form, launches, chain):
    w = _world(pkg.records)
    for asked in ASKED:
        a = dict(_base(w), asked=asked, **(dict(cn=CN, co=CO) if form == "cands" else {}))
        _valid(pkg, ctx, w, fn, a, launches, chain, f"{fn} {form} {asked}")


@pytest.mark.parametrize("fn", SYNC)
def test_second_call_counts_only_its_own_pairs(pkg, ctx, oracle, fn):
    """claim_blocks of a call after another with more claims on the same context: the oracle's, not the sum"""
    w = _world(pkg.records)
    launches, chain = {v[0]: v[2:] for v in VALID if v[1] == "dense"}[fn]
    _valid(pkg, ctx, w, fn, _base(w), launches, chain, f"{fn} first")
    one = dict(_base(w), c=w.c[:1], po=[0, 1], prio=w.prio[:1], n_out=1)
    _valid(pkg, ctx, w, fn, one, launches, chain, f"{fn} second")


# (call, launches of a call with candidates but no pair, with pair_why alone, chain)
NO_PAIRS = [(UNS, 0, {"unsuitable_why"}), (PLACE, 2, {"place", "place_why"}),
            (PRE, 3, {"preempt", "unsuitable_why", "bucket_small"}),
            (PREPL, 6, {"preempt_place", "place_why", "bucket_small"})]
NO_PODS = {UNS: {"unsuitable_why"}, PLACE: set(), PRE: {"preempt", "unsuitable_why"}, PREPL: {"preempt_place", "place_why"}}


@pytest.mark.parametrize("fn,launches,chain", NO_PAIRS)
def test_empty_calls(pkg, ctx, oracle, fn, launches, chain):
    w = _world(pkg.records)
    for asked in (ASKED[0], ASKED[-1]):
        a = dict(_base(w), cn=[], co=[0, 0, 0], asked=asked, null_why=True)        # no pair: pair_why may be NULL
        _load(ctx, w)
        n0 = ctx.launch_count()
        rc, own, why = _raw(pkg, ctx, w, fn, a)
        assert rc == pkg.api.OK, ctx._lib.dra_last_error(ctx._h)
        assert ctx.launch_count() - n0 == launches + (asked[2] or asked[3]), asked
        assert ctx.last_chain() == chain, asked
        pods = dict(_base(w), c=w.c[:0], po=[0], prio=w.prio[:0], n_out=0, asked=asked, null_why=True)
        n0 = ctx.launch_count()
        rc, own, why = _raw(pkg, ctx, w, fn, pods)
        assert rc == pkg.api.OK, ctx._lib.dra_last_error(ctx._h)
        assert ctx.launch_count() == n0 and _untouched(own + why), asked
        assert ctx.last_chain() == NO_PODS[fn], asked


def _plain(ctx, w, fn, cands):
    cn, co = (CN, CO) if cands else (None, None)
    if fn == UNS:
        ctx.unsuitable(w.c, w.po, cn, co)
    elif fn == PLACE:
        ctx.place_pods(w.c, w.po, cn, co)
    elif fn == PRE:
        ctx.preempt(w.c, w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, None, cn, co)
    else:
        ctx.preempt_place(w.c, w.po, w.prio, w.rc, w.rpo, w.rpr, w.ro, None, cn, co)


def _stages(pkg, w, fn, cands, why):
    with pkg.api.Context(device=0) as c:                   # a fresh context: no earlier call's times stand in
        c.set_profiling(True)
        _load(c, w)
        if why:
            rc, _, _ = _raw(pkg, c, w, fn, dict(_base(w), **(dict(cn=CN, co=CO) if cands else {})))
            assert rc == pkg.api.OK
        else:
            _plain(c, w, fn, cands)
        return {k for k, v in c.timings_us().items() if v > 0}


# The stages the reasons calls time where they are known: their walk, after the sort's first stage in the candidate form
TIMED = {(UNS, False): {"bucket_hist"}, (PLACE, False): {"bucket_hist"}, (PLACE, True): {"bucket_hist", "pack"}}


@pytest.mark.parametrize("fn", SYNC)
@pytest.mark.parametrize("cands", [False, True])
def test_profiling_times_the_stages_of_the_plain_call(pkg, oracle, fn, cands):
    w = _world(pkg.records)
    got = _stages(pkg, w, fn, cands, True)
    assert got == _stages(pkg, w, fn, cands, False)
    if (fn, cands) in TIMED:
        assert got == TIMED[fn, cands]


# ---- the sharded calls ------------------------------------------------------------------------------------------------

def _shard(pkg, w, world, why=64, place=8):
    """world contexts serving the two-node inventory of w, rank r node r; why / place: the reservations of
    dra_set_shard_why / dra_set_shard_place made before the export (0: none)"""
    bounds = [0, 1, 2] if world == 2 else [0, 2]
    ctxs = [pkg.api.Context(device=0) for _ in range(world)]
    for r, c in enumerate(ctxs):
        c.comm_init_local(r, world)
        c.set_table(w.t)
        c.set_inventory(w.g, w.off)
        c.set_shard_map(bounds, stray_rank=0)
        if why:
            c.set_shard_why(why)
        if place:
            c.set_shard_place(place)
        if world > 1:
            c.shard_export(64, 0, want_handle=False)
    if world > 1:
        for c in ctxs:
            c.peer_import_local(ctxs)
    return ctxs


class Call:
    """Device inputs of one problem and sentinel-filled device outputs, SLACK elements longer: pod_node, then the four reasons"""

    def __init__(self, pkg, w, c, po, cands):
        import torch
        self.keep = [S.dev(c), S.dev(np.asarray(po, np.uint32))]
        if cands:
            self.keep += [S.dev(np.array(CN, np.uint32)), S.dev(np.array(CO, np.uint32))]
        self.n_claim, self.n_pod = len(c), len(po) - 1
        self.n_pair = int(CO[-1]) if cands else self.n_pod * (len(w.off) - 1)
        self.cands = cands
        sizes = [4 * self.n_pod, self.n_pair, 4 * self.n_pair, 4 * self.n_pod * pkg.api.WHY_N, 4 * self.n_claim]
        self.sizes = sizes
        self.outs = [torch.full((s + 4 * SLACK,), SENTINEL, dtype=torch.uint8, device="cuda:0") for s in sizes]
        torch.cuda.synchronize()                           # (the contexts' streams do not wait for torch's)

    def host(self):
        return [o.cpu().numpy() for o in self.outs]


def _issue(ctx, call, fn, asked=ASKED[-1], null_why=False, flags=0, n_pair=None):
    p = lambda x: None if x is None else C.c_void_p(x)                          # noqa: E731
    d = [t.data_ptr() for t in call.keep]
    cn, co = (p(d[2]), p(d[3])) if call.cands else (None, None)
    o = [t.data_ptr() for t in call.outs]
    wp = [None if (not k or (i == 0 and null_why)) else p(o[1 + i]) for i, k in enumerate(asked)]
    L, h = ctx._lib, ctx._h
    if fn == SU:
        return L.dra_unsuitable_why_batch_global_device(h, p(d[0]), call.n_claim, p(d[1]), call.n_pod, cn, co,
                                                        call.n_pair if n_pair is None else n_pair, *wp, flags)
    n = (call.n_pair if call.cands else 0) if n_pair is None else n_pair
    return L.dra_place_pods_why_batch_global_device(h, p(d[0]), call.n_claim, p(d[1]), call.n_pod, cn, co, n, None,
                                                    call.n_claim, p(o[0]), *wp, flags)


def _shard_refused(pkg, w, ctxs, fn, code, what, **kw):
    for c in ctxs:
        call = Call(pkg, w, w.c, w.po, False)
        n0 = c.launch_count()
        rc = _issue(c, call, fn, **kw)
        assert rc == code, f"{fn} {what}: {rc} (expected {code})"
        c.sync()
        assert c.launch_count() == n0, f"{fn} {what}: launched"
        assert all((h == SENTINEL).all() for h in call.host()), f"{fn} {what}: an output was written"
        assert c.get_inventory().tobytes() == w.g.tobytes(), f"{fn} {what}: live inventory changed"
        c.reset_inventory()
        assert c.get_inventory().tobytes() == w.g.tobytes(), f"{fn} {what}: pristine inventory changed"


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("fn", [SU, SP])
def test_sharded_refusals(pkg, fn, world):
    A = pkg.api
    w = _world(pkg.records)
    cases = [("unknown flag", {}, dict(flags=0x1), A.E_INVAL),
             ("pair_why NULL with pairs", {}, dict(null_why=True), A.E_INVAL),
             ("two faults: unknown flag, pair_why NULL", {}, dict(flags=0x1, null_why=True), A.E_INVAL)]
    if world == 2:
        cases += [("pairs beyond dra_set_shard_why", dict(why=3), {}, A.E_INVAL),
                  ("two faults: no dra_set_shard_why, pair_why NULL", dict(why=0), dict(null_why=True), A.E_STATE),
                  ("two faults: pairs beyond dra_set_shard_why, pair_why NULL", dict(why=3), dict(null_why=True), A.E_INVAL)]
        if fn == SP:
            cases += [("two faults: pods beyond dra_set_shard_place, pair_why NULL", dict(place=1), dict(null_why=True),
                       A.E_STATE)]
    for name, setup, kw, code in cases:
        ctxs = _shard(pkg, w, world, **setup)
        try:
            _shard_refused(pkg, w, ctxs, fn, code, name, **kw)
        finally:
            for c in ctxs:
                c.close()


# (call, form, launches at world 1, at world 2, chain)
SHARD_VALID = [(SU, False, 3, 4, {"unsuitable_why_shard"}), (SU, True, 3, 4, {"unsuitable_why_shard"}),
               (SP, False, 6, 9, {"place_shard", "place_why"}), (SP, True, 7, 10, {"place_shard", "place_why", "bucket_small"})]


def _shard_valid(pkg, w, ctxs, fn, cands, asked, launches, chain, c_, po, what):
    calls = [Call(pkg, w, c_, po, cands) for _ in ctxs]
    before = [c.launch_count() for c in ctxs]
    for c, call in zip(ctxs, calls):
        assert _issue(c, call, fn, asked) == pkg.api.OK, f"{what}: {c._lib.dra_last_error(c._h)}"
    for c in ctxs:
        c.sync()
    cn, co = (np.array(CN, np.uint32), np.array(CO, np.uint32)) if cands else (None, None)
    po = np.asarray(po, np.uint32)
    if fn == SU:
        ref = list(Y.why(w.g, w.off, w.t, c_, po, cn, co, 0))
    else:
        r = PW.place_why(w.g, w.off, w.t, c_, po, cn, co, None, len(c_), 0)
        ref = [r[1]] + list(r[3:])
    dts = [np.uint32, np.uint8, np.uint32, np.uint32, np.uint32]
    for c, call, n0 in zip(ctxs, calls, before):
        assert c.launch_count() - n0 == launches, what
        assert c.last_chain() == chain, what
        h = call.host()
        outs = ([h[0]] if fn == SP else []) + h[1:]
        keys = (["pod_node"] if fn == SP else []) + list(NAMES)
        want = ([True] if fn == SP else []) + list(asked)
        for name, x, y, s, dt, k in zip(keys, outs, ref, call.sizes[-len(keys):], dts[-len(keys):], want):
            if k:
                assert x[:s].view(dt).tobytes() == np.ascontiguousarray(y, dt).ravel().tobytes(), f"{what}: {name}"
                assert (x[s:] == SENTINEL).all(), f"{what}: written past {name}"
            else:
                assert (x == SENTINEL).all(), f"{what}: {name} written without being asked"
        c.set_inventory(w.g, w.off)                        # the next call starts from the loaded inventory


@pytest.mark.parametrize("world", [1, 2])
def test_sharded_valid_calls(pkg, oracle, world):
    w = _world(pkg.records)
    ctxs = _shard(pkg, w, world)
    try:
        for fn, cands, l1, l2, chain in SHARD_VALID:
            for asked in ASKED:
                _shard_valid(pkg, w, ctxs, fn, cands, asked, l1 if world == 1 else l2, chain, w.c, w.po,
                             f"{fn} cands={cands} {asked} world {world}")
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("fn", [SU, SP])
def test_sharded_second_call_counts_only_its_own_pairs(pkg, oracle, fn, world):
    w = _world(pkg.records)
    l1, l2, chain = {(v[0], v[1]): v[2:] for v in SHARD_VALID}[fn, False]
    ctxs = _shard(pkg, w, world)
    try:
        _shard_valid(pkg, w, ctxs, fn, False, ASKED[-1], l1 if world == 1 else l2, chain, w.c, w.po, f"{fn} first")
        _shard_valid(pkg, w, ctxs, fn, False, ASKED[-1], l1 if world == 1 else l2, chain, w.c[:1], [0, 1], f"{fn} second")
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("fn", [SU, SP])
def test_sharded_no_pods(pkg, fn, world):
    """n_pod == 0: nothing exchanged on any rank, no launch, the call's chain"""
    w = _world(pkg.records)
    ctxs = _shard(pkg, w, world)
    try:
        for c in ctxs:
            call = Call(pkg, w, w.c[:0], [0], False)
            n0 = c.launch_count()
            assert _issue(c, call, fn, null_why=True) == pkg.api.OK
            c.sync()
            assert c.launch_count() == n0
            assert c.last_chain() == ({"unsuitable_why_shard"} if fn == SU else set())
            assert all((h == SENTINEL).all() for h in call.host())
    finally:
        for c in ctxs:
            c.close()
