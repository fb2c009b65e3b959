"""GPU suite: preempt and place on a sharded world (dra_preempt_place_batch_global_device, spec §15 "Sharded form").  World
contexts of this process on ONE device, wired as in test_gpu_shard_preempt.py.  Every rank's table, pod_node, pod_status
and evicted_by must be byte for byte the oracle's answer on the world's state (each rank's own node range as that rank
holds it); each rank's own GPU range must end as the oracle's final inventory, and every GPU outside it, and the pristine
copy, must be unchanged."""
import numpy as np
import pytest

import shard_world as S
from shard_world import Running

import preempt_oracle as P
import preempt_place_oracle as PP

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF
SENTINEL = 0x5C


def _slots(pkg, claims):
    """out_off and n_out: slots as if each claim named a node of the inventory"""
    placed = claims.copy()
    placed["node"] = 0
    sl = pkg.records.claim_slots(placed, 1).astype(np.int64)
    return np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32), int(sl.sum())


def _world(pkg, w, world, bounds, invs=None, sizes=(2048, 200000, 2048), n_out_max=65536, place=False, **kw):
    """rank r serving [bounds[r], bounds[r+1]) of the inventory it was given, preempt and place reserved (and place pods
    too, with place=True)"""
    return S.World(pkg, w.table, w.node_off, w.gpus if invs is None else invs, world, bounds, n_out_max=n_out_max,
                   preempt_place=sizes, place=sizes[0] if place else None, **kw)


def _call(W, claims, pod_off, prio, run, cands=None, flags=0, slots=None):
    """slots: (out_off or None, n_out) of the pending claims; None: packed, as _slots lays them out"""
    oo, n_out = _slots(W.pkg, claims) if slots is None else slots
    return S.preempt_place(W, claims, pod_off, prio, run, cands, oo, n_out, flags, SENTINEL)


def _check(W, w, claims, pod_off, prio, run_arrays, run, cands=None, flags=0, what="", slots=None, run_out_off=None):
    """one call against the oracle on the world's state; the ranges, the rest of each copy and the pristine copies.
    Nothing may be written past pod_node, pod_status and evicted_by, nor into evicted_by without pending pods.
    slots as for _call; run_out_off: the running pods' out_off (`run` must carry the same)."""
    before = W.inventories()
    state = W.state()
    cn, co = (None, None) if cands is None else cands
    oo, n_out = _slots(W.pkg, claims) if slots is None else slots
    rc, rpo, rpr, ro = run_arrays
    oracle = lambda fill: PP.preempt_place(state, w.node_off, w.table, claims, pod_off, prio, rc, rpo, rpr,  # noqa: E731
                                           ro, run_out_off, cn, co, oo, n_out,
                                           PP.F_EXHAUSTIVE if flags & W.pkg.api.F_EXHAUSTIVE else 0, fill)
    ref = oracle(SENTINEL)                               # what the call must not write keeps the sentinel
    # the table's slots that no claim owns hold whatever the gathered table held: only the written bytes count
    written = ref[0].view(np.uint8) == oracle(SENTINEL ^ 0xFF)[0].view(np.uint8) if slots is not None else None
    got = _call(W, claims, pod_off, prio, run, cands, flags, (oo, n_out))
    for r, g in enumerate(got):
        for name, x, y in zip(("out", "pod_node", "pod_status", "evicted_by"), g, ref[:4]):
            if name == "out" and written is not None:
                x, y = x.view(np.uint8)[written], y.view(np.uint8)[written]
            if x.tobytes() != y.tobytes():
                bad = np.flatnonzero(x.view(np.uint8) != y.view(np.uint8))[:5]
                pytest.fail(f"{what} rank {r}: {name} differs at bytes {bad}")
        assert "preempt_place_shard" in W.ctxs[r].last_chain()
    W.assert_ranges(before, ref[4], what)
    return ref


def _run_arrays(w):
    return w.run_claims, w.run_pod_off, w.run_prio, w.run_out


def _running(pkg, w):
    return Running(pkg, *_run_arrays(w))


def _cands(form, rng, n_pod, n_node, bounds):
    """candidate lists of one form (None: dense)"""
    if form == "dense":
        return None
    k = 6
    if form == "random":
        nodes = rng.integers(0, n_node + 3, size=n_pod * k)                  # strays included
    elif form == "ascending":
        nodes = np.tile(np.arange(n_node), n_pod)
        k = n_node
    elif form == "descending":
        nodes = np.tile(np.arange(n_node)[::-1], n_pod)
        k = n_node
    elif form == "alternating":                                            # one node of each rank in turn
        world = len(bounds) - 1
        per = [np.arange(bounds[r], bounds[r + 1]) for r in range(world) if bounds[r + 1] > bounds[r]]
        seq = [p[i % len(p)] for i in range(max(len(p) for p in per)) for p in per]
        nodes = np.tile(np.array(seq), n_pod)
        k = len(seq)
    else:                                                                  # duplicates: every node twice in a row
        nodes = np.repeat(rng.integers(0, n_node, size=n_pod * 3), 2)
    return nodes.astype(np.uint32), (np.arange(n_pod + 1) * k).astype(np.uint32)


FORMS = ("dense", "random", "ascending", "descending", "alternating", "duplicates")


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven"), (4, "even"),
                                        (4, "empty")])
@pytest.mark.parametrize("width", [4, 8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    w = pkg.synth.preempt(n_node=16, gpus_per_node=width, n_pending=40, seed=world * 10 + width)
    bounds = S.bounds(S.nn(w), world, kind)
    W = _world(pkg, w, world, bounds)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(world + width)
        statuses = []
        for i, form in enumerate(FORMS):
            flags = pkg.api.F_EXHAUSTIVE if i % 2 else 0
            for r, c in enumerate(W.ctxs):                                   # every call from the inventory as loaded
                c.set_inventory(W.loaded[r], w.node_off)
            ref = _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), run, _cands(form, rng, len(w.prio), S.nn(w), bounds),
                          flags, f"w{world} {kind} width {width} {form} f{flags}")
            statuses.append(ref[2])
        assert (np.concatenate(statuses) == P.EVICT).any()
    finally:
        W.close()


def test_random_forms_and_both_flags(pkg):
    """16 random candidate forms on an uneven world of three ranks, calls chained on the same world."""
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=30, seed=5)
    bounds = S.bounds(S.nn(w), 3, "uneven")
    W = _world(pkg, w, 3, bounds)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(5)
        for i in range(16):
            for r, c in enumerate(W.ctxs):
                c.set_inventory(W.loaded[r], w.node_off)
            _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), run, _cands("random", rng, 30, 20, bounds),
                    pkg.api.F_EXHAUSTIVE * (i % 2), f"random {i}")
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_shared_heavy_world(pkg, world):
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=60, seed=4, mig_nodes=0, shared_per_gpu=12, shapes=("gpu2",))
    W = _world(pkg, w, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for r, c in enumerate(W.ctxs):
                c.set_inventory(W.loaded[r], w.node_off)
            ref = _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), _running(pkg, w), None, flags, f"shared f{flags}")
            assert (ref[2] == P.EVICT).any()
    finally:
        W.close()


def test_selectors_and_long_pods(pkg):
    R = pkg.records
    w = pkg.synth.preempt(n_node=10, gpus_per_node=8, n_pending=30, seed=7)
    attrs = np.zeros(len(w.gpus), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(w.gpus)) % 8
    attrs["mem_total_mib"] = 81920
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 4))])
    c = w.claims.copy()
    mig = c["kind"] == R.KIND_MIG
    c["mem_limit_mib"] = np.where(mig, (np.arange(len(c)) % 4).astype(np.uint32), 0)
    extra = np.zeros(65, R.CLAIM_DTYPE)                      # a pod of 32 1g claims and one of 33
    extra["kind"], extra["count"], extra["profile"] = R.KIND_MIG, 1, R.GI_1_SLICE
    c = np.concatenate([c, extra])
    pod_off = np.concatenate([w.pod_off, [len(w.claims) + 32, len(c)]]).astype(np.uint32)
    prio = np.concatenate([w.prio, [2000, 2000]]).astype(np.int32)
    W = _world(pkg, w, 2, [0, 4, 10], attrs=attrs, sels=sels)
    PP.set_selectors(attrs, sels)
    try:
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for r, ctx in enumerate(W.ctxs):
                ctx.set_inventory(W.loaded[r], w.node_off)
                ctx.set_gpu_attrs(attrs); ctx.set_selectors(sels)
            ref = _check(W, w, c, pod_off, prio, _run_arrays(w), _running(pkg, w), None, flags, f"selectors f{flags}")
            assert ref[2][-1] == P.INVALID
    finally:
        PP.set_selectors()
        W.close()


def test_cfg2_sized_world(pkg):
    """125 nodes of 8 MIG GPUs, 1,000 pending pods, on four ranks: dense and with 8 candidates each."""
    w = pkg.synth.preempt(n_node=125, gpus_per_node=8, n_pending=1000, seed=12, mig_nodes=4)
    bounds = S.bounds(125, 4, "uneven")
    W = _world(pkg, w, 4, bounds, sizes=(1000, 125000, 4096))
    try:
        run = _running(pkg, w)
        _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), run, None, pkg.api.F_EXHAUSTIVE, "cfg2 dense")
        rng = np.random.default_rng(12)
        _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), run, _cands("random", rng, 1000, 125, bounds), 0, "cfg2 chained")
    finally:
        W.close()


def test_world1_equals_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=40, seed=21)
    oo, n_out = _slots(pkg, w.claims)
    W = _world(pkg, w, 1, [0, 12])
    try:
        with pkg.api.Context(device=0) as single:
            for flags in (0, pkg.api.F_EXHAUSTIVE):
                W.ctxs[0].set_inventory(w.gpus, w.node_off)
                got = _call(W, w.claims, w.pod_off, w.prio, _running(pkg, w), None, flags)[0]
                single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
                ref = single.preempt_place(w.claims, w.pod_off, w.prio, *_run_arrays(w), None, None, None, oo, n_out, flags)
                for x, y in zip(got, ref):
                    assert x.tobytes() == y.tobytes()
                assert W.ctxs[0].get_inventory().tobytes() == single.get_inventory().tobytes()
    finally:
        W.close()


def test_equals_place_pods_when_nothing_is_evictable(pkg):
    """No running pod is below any pending pod: the table and the inventory are those of sharded place pods, and so is
    pod_node for every non-empty pod."""
    import torch
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=60, seed=8, prio_lo=500, prio_hi=600, pending_prio=500)
    bounds = S.bounds(20, 3, "uneven")
    oo, n_out = _slots(pkg, w.claims)
    n_pod = len(w.pod_off) - 1
    for flags in (0, pkg.api.F_EXHAUSTIVE):
        A = _world(pkg, w, 3, bounds)
        B = _world(pkg, w, 3, bounds, place=True)
        try:
            got = _call(A, w.claims, w.pod_off, w.prio, _running(pkg, w), None, flags)
            keep = [S.dev(w.claims), S.dev(w.pod_off), S.dev(oo)]
            nodes = [torch.zeros(n_pod, dtype=torch.int32, device="cuda:0") for _ in B.ctxs]
            torch.cuda.synchronize()
            for c, nd in zip(B.ctxs, nodes):
                c.place_pods_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n_pod, None, None, 0,
                                           keep[2].data_ptr(), n_out, nd.data_ptr(), flags)
            for c in B.ctxs:
                c.sync()
            nonempty = np.diff(w.pod_off) > 0
            for r in range(3):
                table = B.ctxs[r].gather_read(np.zeros(n_out, dtype=pkg.records.OUT_DTYPE))
                pn = nodes[r].cpu().numpy().view(np.uint32)
                assert got[r][0].tobytes() == table.tobytes(), f"rank {r} table"
                assert (got[r][1][nonempty] == pn[nonempty]).all() and (got[r][3] == NONE).all()
            assert A.state().tobytes() == B.state().tobytes()
        finally:
            A.close(); B.close()


def test_diverged_copies(pkg):
    """Every rank holds a stale copy of the others' nodes.  dra_preempt_place_batch on one rank answers from its stale
    copy and is wrong; the sharded call answers from the world's state."""
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=40, seed=31)
    stale = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=40, seed=32).gpus
    bounds = [0, 4, 8, 12]
    invs = []
    for r in range(3):
        g = stale.copy()
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        g[a:b] = w.gpus[a:b]
        invs.append(g)
    oo, n_out = _slots(pkg, w.claims)
    W = _world(pkg, w, 3, bounds, invs=invs)
    try:
        assert W.state().tobytes() == w.gpus.tobytes()
        ref = _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), _running(pkg, w), None, 0, "diverged")
        with pkg.api.Context(device=0) as single:
            single.set_table(w.table); single.set_inventory(invs[0], w.node_off)
            one = single.preempt_place(w.claims, w.pod_off, w.prio, *_run_arrays(w), None, None, None, oo, n_out, 0)
        assert any(x.tobytes() != y.tobytes() for x, y in zip(one, ref[:4])), "the stale copy gave the right answer"
    finally:
        W.close()


def test_calls_in_sequence_with_the_inventory_sync(pkg):
    """Calls of changing size chained on one world, interleaved with dra_shard_sync_inventory_device (which shares the
    exchange and its sequence numbers); after each sync every rank's whole inventory is the oracle's."""
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=48, seed=41)
    bounds = S.bounds(16, 3, "uneven")
    W = _world(pkg, w, 3, bounds)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(41)
        for i, (p0, p1) in enumerate(((0, 10), (10, 11), (11, 30), (30, 48))):
            c0, c1 = int(w.pod_off[p0]), int(w.pod_off[p1])
            po = (w.pod_off[p0:p1 + 1] - c0).astype(np.uint32)
            # the running pods stay those of the loaded inventory only in the first call: later calls keep none of them
            if i == 0:
                ra, rr = _run_arrays(w), run
            else:
                z = np.zeros(1, np.uint32)
                ra = (w.run_claims[:0], z, w.run_prio[:0], w.run_out[:0])
                rr = Running(pkg, *ra)
            ref = _check(W, w, w.claims[c0:c1], po, w.prio[p0:p1], ra, rr, _cands("random", rng, p1 - p0, 16, bounds) if i % 2 else None,
                          pkg.api.F_EXHAUSTIVE * (i % 2), f"call {i}")
            for c in W.ctxs:
                c.shard_sync_inventory_device()
            for c in W.ctxs:
                c.sync()
            for r, c in enumerate(W.ctxs):
                assert c.get_inventory().tobytes() == ref[4].tobytes(), f"call {i} rank {r} after the sync"
    finally:
        W.close()


def test_errors(pkg):
    """Host-side refusals return before anything is enqueued.  Each device-detected fault gives DRA_E_INVAL on EVERY rank
    with no output and no inventory word written, the pristine copies untouched, and the next call on the world is right."""
    import torch
    api = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=30, seed=51)
    bounds = [0, 5, 12]
    n_pod = len(w.pod_off) - 1
    oo, n_out = _slots(pkg, w.claims)
    rng = np.random.default_rng(51)
    cn, co = _cands("random", rng, n_pod, 12, bounds)
    d = {k: S.dev(v) for k, v in dict(c=w.claims, po=w.pod_off, pr=w.prio, cn=cn, co=co, oo=oo).items()}
    outs = [torch.full((n_pod * 8 + 4096,), SENTINEL, dtype=torch.uint8, device="cuda:0") for _ in range(3)]
    torch.cuda.synchronize()
    run = _running(pkg, w)

    def raw(c, **k):
        a = dict(c=d["c"].data_ptr(), n_claim=len(w.claims), po=d["po"].data_ptr(), pr=d["pr"].data_ptr(), n_pod=n_pod,
                 cn=d["cn"].data_ptr(), co=d["co"].data_ptr(), n_pair=len(cn), run=run.struct, oo=d["oo"].data_ptr(),
                 n_out=n_out, pn=outs[0].data_ptr(), ps=outs[1].data_ptr(), ev=outs[2].data_ptr(), flags=0)
        a.update(k)
        import ctypes as C
        return c._lib.dra_preempt_place_batch_global_device(c._h, a["c"], a["n_claim"], a["po"], a["pr"], a["n_pod"], a["cn"],
                                                            a["co"], a["n_pair"], C.byref(a["run"]), a["oo"], a["n_out"],
                                                            a["pn"], a["ps"], a["ev"], a["flags"])

    with api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        assert raw(c) == api.E_STATE                                         # no shard
        c.comm_init_local(0, 2); c.set_shard_map(bounds, 0)
        assert raw(c) == api.E_STATE                                         # world 2 without export + import
    W = _world(pkg, w, 2, bounds, sizes=(n_pod, len(cn), len(w.run_prio)))
    try:
        c0 = W.ctxs[0]
        with pytest.raises(api.DraError) as e:
            c0.set_shard_preempt_place(n_pod, len(cn), 8)                    # after the export
        assert e.value.code == api.E_STATE
        assert raw(c0, flags=api.F_FRESH_INVENTORY) == api.E_INVAL
        assert raw(c0, flags=0x80) == api.E_INVAL
        assert raw(c0, n_pod=n_pod + 1) == api.E_INVAL                       # above the reserved sizes
        assert raw(c0, n_pair=len(cn) + 1) == api.E_INVAL
        assert raw(c0, cn=None, co=None, n_pair=0) == api.E_INVAL            # dense: n_pod * n_node pairs > reserved
        big = Running(pkg, np.concatenate([w.run_claims, w.run_claims[:1]]),
                      np.concatenate([w.run_pod_off, [w.run_pod_off[-1] + 1]]).astype(np.uint32),
                      np.concatenate([w.run_prio, w.run_prio[:1]]).astype(np.int32), w.run_out)
        assert raw(c0, run=big.struct) == api.E_INVAL                        # one running pod above the reserved count
        assert raw(c0, n_out=70000) == api.E_INVAL                           # past the exported table
        assert raw(c0, pn=None) == api.E_INVAL
        before = [c.get_inventory() for c in W.ctxs]
        bad_po = w.pod_off.copy(); bad_po[5] = bad_po[7] + 1
        bad_co = co.copy(); bad_co[3] = bad_co[5] + 1
        past = oo.copy(); past[-1] = n_out
        bad_rpo = w.run_pod_off.copy(); bad_rpo[2] = bad_rpo[4] + 1
        two = w.run_out.copy()                                               # a running pod on two nodes
        r0, r1 = int(w.run_pod_off[0]), int(w.run_pod_off[1])
        ok0 = np.flatnonzero((two["status"][r0:r1] == 0))
        far = w.run_out.copy(); far["gpu"][np.flatnonzero(far["status"] == 0)[0]] = len(w.gpus)
        faults = [("pod_off not monotone", dict(po=S.dev(bad_po))), ("cand_off not monotone", dict(co=S.dev(bad_co))),
                  ("slot outside n_out", dict(oo=S.dev(past))),
                  ("running pod_off not monotone", dict(run=Running(pkg, w.run_claims, bad_rpo, w.run_prio, w.run_out))),
                  ("running pod on GPU >= n_gpu", dict(run=Running(pkg, w.run_claims, w.run_pod_off, w.run_prio, far)))]
        if len(ok0):
            g = int(two["gpu"][r0 + ok0[0]])
            two["gpu"][r0 + ok0[0]] = (g + 8) % len(w.gpus)                  # a GPU of another node
            if len(ok0) > 1:
                faults.append(("running pod on two nodes", dict(run=Running(pkg, w.run_claims, w.run_pod_off, w.run_prio, two))))
        for what, k in faults:
            torch.cuda.synchronize()
            for o in outs:
                o.fill_(SENTINEL)
            torch.cuda.synchronize()
            keep = {kk: v for kk, v in k.items()}
            args = {kk: (v.data_ptr() if hasattr(v, "data_ptr") else v.struct if isinstance(v, Running) else v) for kk, v in keep.items()}
            torch.cuda.synchronize()
            for c in W.ctxs:
                assert raw(c, **args) == api.OK, what
            W.wait(api.E_INVAL)
            assert all((o.cpu().numpy() == SENTINEL).all() for o in outs), f"{what}: an output was written"
            for b, c in zip(before, W.ctxs):
                assert c.get_inventory().tobytes() == b.tobytes(), f"{what}: a failed call changed an inventory"
        _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), run, (cn, co), 0, "after the faults")
        for r, c in enumerate(W.ctxs):                                       # the pristine copies are untouched
            c.reset_inventory()
            assert c.get_inventory().tobytes() == w.gpus.tobytes()
    finally:
        W.close()


def test_import_refuses_a_peer_set_up_differently(pkg):
    api = pkg.api
    w = pkg.synth.preempt(n_node=8, gpus_per_node=8, n_pending=8, seed=3)
    ctxs = [api.Context(device=0) for _ in range(2)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, 2); c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard_map([0, 4, 8], 0)
            c.set_shard_preempt_place(64, 512 + r, 64)
            c.shard_export(1024, 0, want_handle=False)
        with pytest.raises(api.DraError) as e:
            ctxs[0].peer_import_local(ctxs)
        assert e.value.code == api.E_INVAL
    finally:
        for c in ctxs:
            c.close()


def test_real_flow_without_a_sync(pkg):
    """The running pods are placed by the sharded pods Allocate on an empty world, with no sync; their OutRecs are the
    gathered table.  Then this call, then dra_shard_sync_inventory_device: every rank's whole inventory is the oracle's."""
    import torch
    from oracle import oracle as O
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=40, seed=61)
    R = pkg.records
    bounds = S.bounds(16, 3, "uneven")
    rsl = R.claim_slots(w.run_claims, 16).astype(np.int64)
    roo = np.concatenate([[0], np.cumsum(rsl)[:-1]]).astype(np.uint32)
    rn_out = int(rsl.sum())
    W = _world(pkg, w, 3, bounds, invs=[w.empty] * 3)
    try:
        dc, dp, do = S.dev(w.run_claims), S.dev(w.run_pod_off), S.dev(roo)
        torch.cuda.synchronize()
        for c in W.ctxs:
            c.allocate_pods_global_device(dc.data_ptr(), len(w.run_claims), dp.data_ptr(), len(w.run_pod_off) - 1,
                                          do.data_ptr(), rn_out, 0)
        for c in W.ctxs:
            c.sync()
        ref_out, ref_inv = O.allocate_pods(w.empty, w.node_off, w.table, w.run_claims, w.run_pod_off, roo, rn_out, 0)
        tables = [c.gather_read(np.zeros(rn_out, dtype=R.OUT_DTYPE)) for c in W.ctxs]
        assert all(t.tobytes() == ref_out.tobytes() for t in tables)
        assert W.state().tobytes() == ref_inv.tobytes()
        ra = (w.run_claims, w.run_pod_off, w.run_prio, tables[0])
        run = Running(pkg, *ra, out_off=roo)
        oo, n_out = _slots(pkg, w.claims)
        ref = PP.preempt_place(ref_inv, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                               w.run_prio, tables[0], roo, None, None, oo, n_out, PP.F_EXHAUSTIVE)
        got = _call(W, w.claims, w.pod_off, w.prio, run, None, pkg.api.F_EXHAUSTIVE)
        for r, g in enumerate(got):
            for x, y in zip(g, ref[:4]):
                assert x.tobytes() == y.tobytes(), f"rank {r}"
        assert (ref[2] == P.EVICT).any()
        for c in W.ctxs:
            c.shard_sync_inventory_device()
        for c in W.ctxs:
            c.sync()
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == ref[4].tobytes(), f"rank {r} after the sync"
    finally:
        W.close()


def test_interleaved_with_the_gathering_calls(pkg):
    """Sharded place pods and pods Allocate, whose tables travel as packets, before and after this call on the same world
    (the result tables share the exported region and its parity): every call against its oracle on the world's state."""
    import torch
    import place_oracle as PL
    from oracle import oracle as O
    R = pkg.records
    w = pkg.synth.preempt(n_node=16, gpus_per_node=8, n_pending=48, seed=71)
    bounds = S.bounds(16, 3, "uneven")
    W = _world(pkg, w, 3, bounds, place=True)
    try:
        run = _running(pkg, w)
        for i in range(3):
            p0, p1 = 16 * i, 16 * i + 16
            c0, c1 = int(w.pod_off[p0]), int(w.pod_off[p1])
            claims = w.claims[c0:c1]
            po = (w.pod_off[p0:p1 + 1] - c0).astype(np.uint32)
            oo, n_out = _slots(pkg, claims)
            # place pods
            state = W.state()
            ref_out, ref_node, ref_inv = PL.place_pods(state, w.node_off, w.table, claims, po, None, None, oo, n_out, 0)
            keep = [S.dev(claims), S.dev(po), S.dev(oo)]
            nodes = [torch.zeros(16, dtype=torch.int32, device="cuda:0") for _ in W.ctxs]
            torch.cuda.synchronize()
            for c, nd in zip(W.ctxs, nodes):
                c.place_pods_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), 16, None, None, 0,
                                           keep[2].data_ptr(), n_out, nd.data_ptr(), 0)
            for c in W.ctxs:
                c.sync()
            for c in W.ctxs:
                assert c.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE)).tobytes() == ref_out.tobytes(), f"place {i}"
            assert W.state().tobytes() == ref_inv.tobytes()
            # this call, on the same pods again (they now compete with their own placements)
            _check(W, w, claims, po, w.prio[p0:p1], _run_arrays(w), run, None, pkg.api.F_EXHAUSTIVE * (i % 2), f"preempt place {i}")
            # pods Allocate of the same pods on the nodes place pods chose
            pc = claims.copy()
            for p in range(16):
                pc["node"][po[p]:po[p + 1]] = ref_node[p] if ref_node[p] != NONE else 0
            state = W.state()
            ref_out2, ref_inv2 = O.allocate_pods(state, w.node_off, w.table, pc, po, oo, n_out, 0)
            keep2 = [S.dev(pc), S.dev(po), S.dev(oo)]
            torch.cuda.synchronize()
            for c in W.ctxs:
                c.allocate_pods_global_device(keep2[0].data_ptr(), len(pc), keep2[1].data_ptr(), 16, keep2[2].data_ptr(), n_out, 0)
            for c in W.ctxs:
                c.sync()
            for c in W.ctxs:
                assert c.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE)).tobytes() == ref_out2.tobytes(), f"pods Allocate {i}"
            assert W.state().tobytes() == ref_inv2.tobytes()
    finally:
        W.close()


def test_a_late_peer_fails_the_call_on_every_rank(pkg, monkeypatch):
    """Ranks 0 and 1 are enqueued, rank 2 only after their exchange has timed out.  Rank 2 receives every range, but the
    verdict agreement fails the call on every rank with DRA_E_NCCL, nothing is written anywhere, and the next call on the
    same world is right."""
    import time
    import torch
    monkeypatch.setenv("DRA_PEER_TIMEOUT_MS", "200")                  # read by the export
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=24, seed=81)
    W = _world(pkg, w, 3, [0, 4, 8, 12])
    try:
        run = _running(pkg, w)
        n_pod = len(w.pod_off) - 1
        oo, n_out = _slots(pkg, w.claims)
        keep = [S.dev(w.claims), S.dev(w.pod_off), S.dev(w.prio), S.dev(oo)]
        outs = [[torch.full((s + S.PAD,), SENTINEL, dtype=torch.uint8, device="cuda:0") for s in (n_pod * 4, n_pod, len(w.run_prio) * 4)]
                for _ in W.ctxs]
        before = [c.get_inventory() for c in W.ctxs]
        torch.cuda.synchronize()
        for r, (c, o) in enumerate(zip(W.ctxs, outs)):
            if r == 2:
                time.sleep(1.5)                                        # well past the 200 ms the others wait
            c.preempt_place_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                          None, None, 0, run.struct, keep[3].data_ptr(), n_out,
                                          o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), 0)
        W.wait(pkg.api.E_NCCL)
        for r, (c, o) in enumerate(zip(W.ctxs, outs)):
            assert all((t.cpu().numpy() == SENTINEL).all() for t in o), f"rank {r} wrote an output"
            assert c.get_inventory().tobytes() == before[r].tobytes(), f"rank {r} wrote its inventory"
        _check(W, w, w.claims, w.pod_off, w.prio, _run_arrays(w), run, None, 0, "after the late peer")
    finally:
        W.close()
