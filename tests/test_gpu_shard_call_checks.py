"""GPU suite: what the sharded pod calls (UnsuitableNodes, pods Allocate, place pods, preemption, pod capacity, preempt and
place) and the inventory sync promise about their arguments and their world.  World contexts of this process on ONE
device, wired with dra_comm_init_local / dra_peer_import_local, called through the raw ABI on sentinel-filled device
outputs.  A refused call returns its code with no output byte written, no live or pristine inventory word changed and no
kernel launched.  A call refused on the host is issued only on the ranks that refuse it, so no peer ever waits for it.
A valid call of each, issued on every rank, launches the kernels it is known for and reports its chain."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_pod_call_checks import _world
import shard_world as S

pytestmark = pytest.mark.gpu
SENTINEL = 0xA7
U, A, P, R, K, PP, SYNC = "unsuitable", "allocate_pods", "place_pods", "preempt", "capacity", "preempt_place", "sync"
POD_CALLS = (U, A, P, R, K, PP)
FRESH = 0x2                                                # DRA_F_FRESH_INVENTORY
OUT_BYTES = 256                                            # each output buffer, sentinel-filled


def _setup(pkg, w, world, shard="map", export=True, sizes=True, inv=True, n_out_max=64):
    """world contexts serving the two-node inventory of w, rank r node r.  shard: "map", "bare" (dra_set_shard) or None;
    sizes: the five setters called before the export (False: none); inv False: a world of 2 whose inventory and map are
    loaded after the export, so no staging was reserved for it."""
    bounds = [0, 1, 2] if world == 2 else [0, 2]
    if inv:
        sz = dict(pairs=64, place=8, preempt=(8, 64, 8), capacity=64, preempt_place=(8, 64, 8)) if sizes else {}
        return S.World(pkg, w.t, w.off, w.g, world, None if shard is None else bounds, bare=shard == "bare", export=export,
                       n_out_max=n_out_max, **sz).ctxs
    ctxs = [pkg.api.Context(device=0) for _ in range(world)]
    for r, c in enumerate(ctxs):
        c.comm_init_local(r, world)
        c.set_table(w.t)
        c.set_shard_pairs(64); c.set_shard_place(8); c.set_shard_preempt(8, 64, 8); c.set_shard_capacity(64)
        c.set_shard_preempt_place(8, 64, 8)
        c.shard_export(n_out_max, 0, want_handle=False)
        c.set_inventory(w.g, w.off)
        c.set_shard_map(bounds, stray_rank=0)
    for c in ctxs:
        c.peer_import_local(ctxs)
    return ctxs


def _close(ctxs):
    for c in ctxs:
        c.close()


class Call:
    """The device inputs of the base problem and sentinel-filled device outputs for one call"""

    def __init__(self, pkg, w):
        import torch
        c = w.c.copy()
        c["node"] = [0, 1]                                 # pods Allocate: each pod names its node
        self.keep = {"c": S.dev(w.c), "ca": S.dev(c), "po": S.dev(w.po), "prio": S.dev(w.prio), "cn": S.dev(np.array([0, 1, 1], np.uint32)),
                     "co": S.dev(np.array([0, 2, 3], np.uint32))}
        self.run_keep = [S.dev(w.rc), S.dev(w.rpo), S.dev(w.rpr), S.dev(w.ro)]
        self.run = pkg.api.RunningPods(self.run_keep[0].data_ptr(), len(w.rc), self.run_keep[1].data_ptr(), len(w.rpo) - 1,
                                       self.run_keep[2].data_ptr(), None, self.run_keep[3].data_ptr(), len(w.ro))
        self.outs = [torch.full((OUT_BYTES,), SENTINEL, dtype=torch.uint8, device="cuda:0") for _ in range(6)]
        self.n_claim, self.n_pod = len(w.c), len(w.po) - 1
        torch.cuda.synchronize()                           # (the contexts' streams do not wait for torch's)

    def untouched(self):
        return all((o.cpu().numpy() == SENTINEL).all() for o in self.outs)


def _p(x):
    return None if x is None else C.c_void_p(x)


def _issue(ctx, call, fn, **kw):
    """dra_<fn> through ctypes on call's buffers; kw overrides the base arguments (None: a NULL pointer).  Returns the code."""
    d = lambda k: call.keep[k].data_ptr()                  # noqa: E731
    o = [t.data_ptr() for t in call.outs]
    a = dict(claims=d("ca") if fn == A else d("c"), n_claim=call.n_claim, pod_off=d("po"), prio=d("prio"), n_pod=call.n_pod,
             cn=None, co=None, n_pair=None, out_off=None, n_out=call.n_claim, flags=0, running=C.byref(call.run),
             o0=o[0], o1=o[1], o2=o[2], o3=o[3], o4=o[4], o5=o[5], max_victims=4, max_copies=4)
    if kw.get("cands"):
        a.update(cn=d("cn"), co=d("co"), n_pair=3)
    kw.pop("cands", None)
    a.update(kw)
    if a["n_pair"] is None:                                # the dense form's pairs
        a["n_pair"] = a["n_pod"] * 2 if fn in (U, R, K) else 0
    L, h = ctx._lib, ctx._h
    if fn == U:
        return L.dra_unsuitable_batch_global_device(h, _p(a["claims"]), a["n_claim"], _p(a["pod_off"]), a["n_pod"], _p(a["cn"]),
                                                    _p(a["co"]), a["n_pair"], _p(a["o0"]), a["flags"])
    if fn == A:
        return L.dra_allocate_pods_batch_global_device(h, _p(a["claims"]), a["n_claim"], _p(a["pod_off"]), a["n_pod"],
                                                       _p(a["out_off"]), a["n_out"], a["flags"])
    if fn == P:
        return L.dra_place_pods_batch_global_device(h, _p(a["claims"]), a["n_claim"], _p(a["pod_off"]), a["n_pod"], _p(a["cn"]),
                                                    _p(a["co"]), a["n_pair"], _p(a["out_off"]), a["n_out"], _p(a["o0"]), a["flags"])
    if fn == R:
        return L.dra_preempt_batch_global_device(h, _p(a["claims"]), a["n_claim"], _p(a["pod_off"]), _p(a["prio"]), a["n_pod"],
                                                 _p(a["cn"]), _p(a["co"]), a["n_pair"], a["running"], _p(a["o0"]), _p(a["o1"]),
                                                 _p(a["o2"]), _p(a["o3"]), _p(a["o4"]), _p(a["o5"]), a["max_victims"], a["flags"])
    if fn == K:
        return L.dra_pod_capacity_batch_global_device(h, _p(a["claims"]), a["n_claim"], _p(a["pod_off"]), a["n_pod"], _p(a["cn"]),
                                                      _p(a["co"]), a["n_pair"], a["max_copies"], _p(a["o0"]), _p(a["o1"]),
                                                      _p(a["o2"]), _p(a["o3"]), a["flags"])
    if fn == PP:
        return L.dra_preempt_place_batch_global_device(h, _p(a["claims"]), a["n_claim"], _p(a["pod_off"]), _p(a["prio"]),
                                                       a["n_pod"], _p(a["cn"]), _p(a["co"]), a["n_pair"], a["running"],
                                                       _p(a["out_off"]), a["n_out"], _p(a["o0"]), _p(a["o1"]), _p(a["o2"]),
                                                       a["flags"])
    return L.dra_shard_sync_inventory_device(h)


def _refused(pkg, w, ctx, fn, code, what, **kw):
    """fn refused on ctx's host with code: nothing launched, no output byte and no live or pristine inventory word written"""
    call = Call(pkg, w)
    n0 = ctx.launch_count()
    rc = _issue(ctx, call, fn, **kw)
    assert rc == code, f"{fn} {what}: {rc} (expected {code}): {ctx._lib.dra_last_error(ctx._h)}"
    ctx.sync()
    assert ctx.launch_count() == n0, f"{fn} {what}: launched"
    assert call.untouched(), f"{fn} {what}: an output was written"
    assert ctx.get_inventory().tobytes() == w.g.tobytes(), f"{fn} {what}: live inventory changed"
    ctx.reset_inventory()
    assert ctx.get_inventory().tobytes() == w.g.tobytes(), f"{fn} {what}: pristine inventory changed"


BIG = 0xFFFFFFF1
# (name, calls, arguments, code): one bad argument each, except the rows marked "two faults", which pin the order of the
# checks
ARG_CASES = [
    ("pod_off NULL", POD_CALLS, dict(pod_off=None), "INVAL"),
    ("claims NULL with claims", POD_CALLS, dict(claims=None), "INVAL"),
    ("unknown flag", POD_CALLS, dict(flags=0x1), "INVAL"),
    ("FRESH where not taken", (U, R, K, PP), dict(flags=FRESH), "INVAL"),
    ("cand_nodes without cand_off", (U, P, R, K, PP), dict(cands=True, co=None), "INVAL"),
    ("cand_off without cand_nodes", (U, P, R, K, PP), dict(cands=True, cn=None), "INVAL"),
    ("dense n_pair != n_pod x n_node", (U, R, K), dict(n_pair=3), "INVAL"),
    ("dense n_pair != 0", (P, PP), dict(n_pair=1), "INVAL"),
    ("more than 0xFFFFFFF0 pairs", (U, P, R, K, PP), dict(cands=True, n_pair=BIG), "INVAL"),
    ("bits NULL with pairs", (U,), dict(o0=None), "INVAL"),
    ("pod_node NULL with pods", (P, PP), dict(o0=None), "INVAL"),
    ("prio NULL with pods", (R, PP), dict(prio=None), "INVAL"),
    ("running NULL", (R, PP), dict(running=None), "INVAL"),
    ("pod_status NULL with pods", (R,), dict(o3=None), "INVAL"),
    ("max_victims without victims", (R,), dict(o5=None), "INVAL"),
    ("pair_copies NULL with pairs", (K,), dict(o0=None), "INVAL"),
    ("max_copies 0", (K,), dict(max_copies=0), "INVAL"),
    ("evicted_by NULL with running pods", (PP,), dict(o2=None), "INVAL"),
    ("n_out < n_claim without out_off", (A, P, PP), dict(n_out=1), "INVAL"),
    ("two faults: unknown flag, dense n_pair", (U, R, K), dict(flags=0x1, n_pair=3), "INVAL"),
    ("two faults: n_out, dense n_pair", (P, PP), dict(n_out=1, n_pair=1), "INVAL"),
]


@pytest.mark.parametrize("world", [1, 2])
def test_argument_refusals(pkg, world):
    A_ = pkg.api
    w = _world(pkg.records)
    ctxs = _setup(pkg, w, world)
    try:
        for name, fns, kw, code in ARG_CASES:
            for fn in fns:
                for c in ctxs:
                    _refused(pkg, w, c, fn, getattr(A_, "E_" + code), name, **kw)
    finally:
        _close(ctxs)


# (name, calls, world, setup: the keyword arguments of _setup, arguments, code): the state a call needs
STATE_CASES = [
    ("no dra_set_shard", (U, A, P, K, PP), 1, dict(shard=None), {}, "STATE"),
    ("no dra_set_shard_map at world > 1", (A, P, R, K, PP, SYNC), 2, dict(shard="bare"), {}, "STATE"),
    ("no export at world > 1", POD_CALLS + (SYNC,), 2, dict(export=False), {}, "STATE"),
    ("no exchange reserved", (K, PP), 2, dict(sizes=False), {}, "STATE"),
    ("no exchange reserved, no pairs", (K,), 2, dict(sizes=False), dict(cands=True, n_pair=0), "STATE"),
    ("no pairs reserved", (U, R), 2, dict(sizes=False), {}, "INVAL"),
    ("no pods reserved", (P,), 2, dict(sizes=False), {}, "STATE"),
    ("inventory loaded after the export", (PP, SYNC), 2, dict(inv=False), {}, "STATE"),
    ("n_out beyond the exported table", (A, P, PP), 2, dict(n_out_max=1), dict(n_out=2), "INVAL"),
    ("two faults: no map, n_out beyond the table", (A, P), 2, dict(shard="bare", n_out_max=1), dict(n_out=2), "STATE"),
    ("two faults: n_out beyond the table, no pods reserved", (P,), 2, dict(sizes=False, n_out_max=1), dict(n_out=2), "INVAL"),
    ("two faults: no exchange reserved, n_out beyond the table", (PP,), 2, dict(sizes=False, n_out_max=1), dict(n_out=2), "STATE"),
    ("two faults: no exchange reserved, too many pairs", (K,), 2, dict(sizes=False), dict(cands=True, n_pair=BIG), "INVAL"),
    ("two faults: no map, no pairs reserved", (R, K), 2, dict(shard="bare", sizes=False), {}, "STATE"),
    ("two faults: unknown flag, no export", POD_CALLS, 2, dict(export=False), dict(flags=0x1), "INVAL"),
]


@pytest.mark.parametrize("case", STATE_CASES, ids=[c[0] for c in STATE_CASES])
def test_state_refusals(pkg, case):
    name, fns, world, setup, kw, code = case
    A_ = pkg.api
    w = _world(pkg.records)
    ctxs = _setup(pkg, w, world, **setup)
    try:
        for fn in fns:
            for c in ctxs:
                _refused(pkg, w, c, fn, getattr(A_, "E_" + code), name, **kw)
    finally:
        _close(ctxs)


def test_sizes_beyond_the_reservation(pkg):
    """Each exchange reserved one size too small: place pods refuses with DRA_E_STATE, the others with DRA_E_INVAL"""
    A_ = pkg.api
    w = _world(pkg.records)
    for fn, setter, args, code in ((U, "set_shard_pairs", (3,), A_.E_INVAL), (P, "set_shard_place", (1,), A_.E_STATE),
                                   (R, "set_shard_preempt", (1, 64, 8), A_.E_INVAL), (R, "set_shard_preempt", (8, 3, 8), A_.E_INVAL),
                                   (R, "set_shard_preempt", (8, 64, 3), A_.E_INVAL), (K, "set_shard_capacity", (3,), A_.E_INVAL),
                                   (PP, "set_shard_preempt_place", (1, 64, 8), A_.E_INVAL),
                                   (PP, "set_shard_preempt_place", (8, 3, 8), A_.E_INVAL),
                                   (PP, "set_shard_preempt_place", (8, 64, 1), A_.E_INVAL)):
        ctxs = _setup(pkg, w, 2, export=False)
        try:
            for c in ctxs:
                getattr(c, setter)(*args)
                c.shard_export(64, 0, want_handle=False)
            for c in ctxs:
                c.peer_import_local(ctxs)
            for c in ctxs:
                _refused(pkg, w, c, fn, code, f"{setter}{args}")
            with pytest.raises(A_.DraError) as e:                      # every setter: only before the export
                getattr(ctxs[0], setter)(*args)
            assert e.value.code == A_.E_STATE
        finally:
            _close(ctxs)


def test_world_one_preemption_needs_no_shard(pkg):
    """dra_preempt_batch_global_device at world 1 runs on [0, n_node) without dra_set_shard; the other calls refuse"""
    w = _world(pkg.records)
    ctxs = _setup(pkg, w, 1, shard=None)
    try:
        call = Call(pkg, w)
        assert _issue(ctxs[0], call, R) == pkg.api.OK
        ctxs[0].sync()
        assert not call.untouched()
    finally:
        _close(ctxs)


def test_inventory_changes_after_the_export(pkg):
    """A shard map no longer spanning the inventory, and an inventory grown past the sync's staging"""
    A_ = pkg.api
    w = _world(pkg.records)
    g3, off3 = pkg.records.make_inventory([1, 1, 1], mig=True)
    ctxs = _setup(pkg, w, 2)
    try:
        for c in ctxs:
            c.set_inventory(g3, off3)
        w3 = type(w)(**dict(vars(w), g=g3, off=off3))
        for fn in (R, K, PP, SYNC):
            for c in ctxs:
                _refused(pkg, w3, c, fn, A_.E_STATE, "map not spanning the inventory", **(dict(n_pair=6) if fn in (R, K) else {}))
    finally:
        _close(ctxs)


# (call, form, launches at world 1, at world 2, chain: None where the call leaves the chain as it was)
VALID = [
    (U, "dense", 3, 4, None), (U, "cands", 3, 4, None),
    (A, "dense", 4, 5, {"pod_shard", "bucket_small"}),
    (P, "dense", 4, 6, {"place_shard"}), (P, "cands", 5, 7, {"place_shard", "bucket_small"}),
    (R, "dense", 8, 9, {"preempt_shard", "bucket_small"}), (R, "cands", 8, 9, {"preempt_shard", "bucket_small"}),
    (K, "dense", 3, 4, {"pod_capacity_shard"}), (K, "cands", 3, 4, {"pod_capacity_shard"}),
    (PP, "dense", 6, 9, {"preempt_place_shard", "bucket_small"}), (PP, "cands", 7, 10, {"preempt_place_shard", "bucket_small"}),
    (SYNC, "-", 0, 2, None),
]


@pytest.mark.parametrize("world", [1, 2])
def test_valid_calls(pkg, world):
    """Each call on every rank (enqueued on all before any waits): its launches and its chain bits"""
    w = _world(pkg.records)
    ctxs = _setup(pkg, w, world)
    try:
        for fn, form, l1, l2, chain in VALID:
            calls = [Call(pkg, w) for _ in ctxs]
            before = [(c.last_chain(), c.launch_count()) for c in ctxs]
            for c, call in zip(ctxs, calls):
                assert _issue(c, call, fn, cands=form == "cands") == pkg.api.OK, (fn, form, c._lib.dra_last_error(c._h))
            for c in ctxs:
                c.sync()
            for c, (ch, n0) in zip(ctxs, before):
                assert c.launch_count() - n0 == (l1 if world == 1 else l2), (fn, form, world)
                if fn == A and world == 2:
                    assert c.last_chain() == chain | {"pod_gather"}, (fn, form)
                else:
                    assert c.last_chain() == (ch if chain is None else chain), (fn, form, world)
            for c in ctxs:                                 # the next call starts from the loaded inventory
                c.set_inventory(w.g, w.off)
    finally:
        _close(ctxs)
