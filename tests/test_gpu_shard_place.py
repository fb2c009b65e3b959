"""GPU suite: place pods on a sharded world (dra_place_pods_batch_global_device).  World contexts of this process on ONE
device, wired like test_gpu_shard_pods.py.  Every rank's whole table and pod_node must be byte for byte the §13 oracle's
answer on the world's real state (the inventory each rank holds for its own node range), each rank's own GPU range the
oracle's inventory afterwards, and no rank may write GPUs outside its range."""
from types import SimpleNamespace

import numpy as np
import pytest

from test_place_pods import NONE, _flat, placed_offsets

import place_oracle as P
import shard_world as S

pytestmark = pytest.mark.gpu
MAX_PODS = 4096
N_OUT_MAX = 1 << 16


def _flags(api):
    return [0, api.F_EXHAUSTIVE, api.F_FRESH_INVENTORY, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY]


def _world(pkg, w, world, bounds, stray_rank=0, max_pods=MAX_PODS, attrs=None, sels=None, cap_per_rank=0, max_pairs=None):
    """every rank holding the whole inventory, with room for the replicated pod states reserved before the export"""
    return S.World(pkg, w.table, w.node_off, w.gpus, world, bounds, stray_rank, attrs, sels, n_out_max=N_OUT_MAX,
                   cap_per_rank=cap_per_rank, pairs=max_pairs, place=max_pods)


def _place(W, claims, pod_off, cn, co, out_off, n_out, flags=0):
    """every rank's whole table and pod_node"""
    res = S.place(W, claims, pod_off, None if co is None else (cn, co), out_off, n_out, flags)
    return [t for t, _ in res], [n for _, n in res]


def _check(W, w, claims, pod_off, cn, co, out_off, n_out, flags, what):
    """One call against the §13 oracle on the world's state: every rank's table and pod_node, its own range the oracle's,
    nothing written outside it, the chain taken."""
    api = W.pkg.api
    before = W.inventories()
    src = w.gpus if flags & api.F_FRESH_INVENTORY else W.state()
    ref, ref_node, ref_inv = P.place_pods(src, w.node_off, w.table, claims, pod_off, cn, co, out_off, n_out,
                                          P.F_EXHAUSTIVE if flags & api.F_EXHAUSTIVE else 0)
    tables, nodes = _place(W, claims, pod_off, cn, co, out_off, n_out, flags)
    S.same_tables(tables, ref, what)
    for r in range(W.world):
        assert nodes[r].tobytes() == ref_node.tobytes(), f"{what}: rank {r} pod_node differs"
    W.assert_ranges(before, ref_inv, what)
    assert "place_shard" in W.ctxs[0].last_chain()
    return ref, ref_node


def _forms(rng, n_pod, n_node, bounds):
    """Candidate forms: the dense form, 8 random (some naming no node, NONE), every node ascending, every node descending
    (every pod crosses the ranks backwards), alternating between the ranks' ranges, duplicates and zero-candidate pods."""
    k = 8
    rand = rng.integers(0, n_node + 3, size=n_pod * k).astype(np.uint32)
    rand[5::k] = NONE
    asc = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
    every = (np.arange(n_pod + 1) * n_node).astype(np.uint32)
    ranges = [np.arange(bounds[r], bounds[r + 1]) for r in range(len(bounds) - 1) if bounds[r + 1] > bounds[r]]
    alt = [x for group in zip(*[np.resize(g, n_node) for g in ranges]) for x in group][:n_node]
    per = rng.integers(0, 6, n_pod); per[::5] = 0
    dup = [list(rng.integers(0, n_node, m)) * 2 for m in per]
    return {"dense": (None, None), "random8": (rand, (np.arange(n_pod + 1) * k).astype(np.uint32)),
            "ascending": (asc, every), "descending": (asc[::-1].copy(), every),
            "alternating": (np.tile(np.array(alt, dtype=np.uint32), n_pod), every), "duplicates": _flat(dup)}


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_matches_oracle(pkg, world):
    """Every candidate form on even, uneven and empty ranges; the flag combinations one after the other on one world."""
    rng = np.random.default_rng(world)
    kind = ["even", "uneven", "empty", "uneven"][world - 1]
    w, pod_off = pkg.synth.pods(500, 23, 100 + world)
    n_pod = len(pod_off) - 1
    bounds = S.bounds(w.n_node, world, kind)
    W = _world(pkg, w, world, bounds, world - 1)
    try:
        for i, (name, (cn, co)) in enumerate(_forms(rng, n_pod, w.n_node, bounds).items()):
            flags = _flags(pkg.api)[i % 4]
            ref, ref_node = _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), flags, f"{name} flags {flags}")
            if name != "duplicates":
                assert (ref_node != NONE).any() and (ref_node == NONE).any(), name
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_flags_in_sequence(pkg, world):
    """All four flag combinations one call after another, twice over, so call sequence numbers and table parities advance;
    stale-call state words must lose to the current call's."""
    rng = np.random.default_rng(7 + world)
    w, pod_off = pkg.synth.pods(400, 17, 60 + world)
    n_pod = len(pod_off) - 1
    bounds = S.bounds(w.n_node, world, "uneven")
    W = _world(pkg, w, world, bounds, 0)
    try:
        for rep in range(2):
            for flags in _flags(pkg.api):
                cn = rng.integers(0, w.n_node, n_pod * 6).astype(np.uint32)
                co = (np.arange(n_pod + 1) * 6).astype(np.uint32)
                _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), flags, f"rep {rep} flags {flags}")
    finally:
        W.close()


@pytest.mark.parametrize("world", [1, 3])
def test_mixed_pods(pkg, world):
    """Pods cut from synth.mixed with selectors: empty pods, a pod of more than 32 claims, malformed claims, GPU claims of
    count > 1 (out_off), random candidates across ranks."""
    api = pkg.api
    rng = np.random.default_rng(30 + world)
    w = pkg.synth.mixed(2400, 31, 70 + world, invalid=True)
    attrs, sels = pkg.synth.with_selectors(w, world)
    bounds = S.bounds(w.n_node, world, "even")
    claims, pod_off, _, _ = S.malformed_mixed(pkg, w, bounds, rng, False)
    out_off, n_out = placed_offsets(pkg.records, claims, w.n_node)
    n_pod = len(pod_off) - 1
    cn = rng.integers(0, w.n_node + 2, n_pod * 5).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 5).astype(np.uint32)
    W = _world(pkg, w, world, bounds, 0, attrs=attrs, sels=sels)
    P.set_selectors(attrs, sels)
    try:
        for flags in (0, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY):
            for c_, o_ in ((cn, co), (None, None)):
                ref, _ = _check(W, w, claims, pod_off, c_, o_, out_off, int(n_out), flags, f"mixed flags {flags}")
                assert (ref["status"] == pkg.records.ST_INVALID).any()
    finally:
        P.set_selectors()
        W.close()


def test_search_limit_survives_a_hand_off(pkg):
    """7 x 1g + 7g: the exhaustive search runs out of budget on the empty GPU of node 0 (rank 0); node 1 (rank 1) is full
    and fails the pod with POD.  The limit bit rides in the state word to rank 1, whose records must say SEARCH_LIMIT."""
    R, api = pkg.records, pkg.api
    from test_pod_mode import _mig
    g, off = R.make_inventory([1, 1, 1], mig=True)
    g["busy"][1] = 0xFF
    w = SimpleNamespace(gpus=g, node_off=off, table=R.default_table(), n_node=3)
    c = _mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE])
    pod_off = np.array([0, 8], np.uint32)
    W = _world(pkg, w, 3, [0, 1, 2, 3], 2)
    try:
        for cands in ([0, 1], [1, 0], [0, 1, 2], [2, 1, 0]):
            cn, co = _flat([cands])
            ref, node = _check(W, w, c, pod_off, cn, co, None, 8, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY, f"cands {cands}")
            assert set(ref["status"]) == {R.ST_SEARCH_LIMIT} and list(node) == [NONE]
        cn, co = _flat([[0, 1]])
        ref, _ = _check(W, w, c, pod_off, cn, co, None, 8, api.F_FRESH_INVENTORY, "first-fit")
        assert set(ref["status"]) == {R.ST_POD}
    finally:
        W.close()


def test_windows_wider_than_the_resident_warps(pkg):
    """10,000 nodes over two ranks on one device: each rank's walk takes its whole share of the residency while the peer
    still sorts its 80,000 pairs with the CTA-wide histogram, and each warp cycles over several nodes."""
    rng = np.random.default_rng(21)
    w, pod_off = pkg.synth.pods(10_000, 10_000, 21)
    n_pod = len(pod_off) - 1
    cn = rng.integers(0, w.n_node + 2, n_pod * 8).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 8).astype(np.uint32)
    W = _world(pkg, w, 2, [0, 5000, 10_000], 0, max_pods=n_pod)
    try:
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), flags, f"10k nodes flags {flags}")
    finally:
        W.close()


def test_single_candidate_equals_sharded_pods_allocate(pkg):
    """One candidate per pod, the node its claims name: the table equals dra_allocate_pods_batch_global_device's."""
    api = pkg.api
    w, pod_off = pkg.synth.pods(600, 20, 9)
    first = w.claims["node"][pod_off[:-1]].astype(np.uint32)
    co = np.arange(len(pod_off), dtype=np.uint32)
    W = _world(pkg, w, 3, S.bounds(w.n_node, 3, "uneven"), 1)
    try:
        for flags in (api.F_FRESH_INVENTORY, api.F_FRESH_INVENTORY | api.F_EXHAUSTIVE):
            ref = S.pods(W, w.claims, pod_off, None, len(w.claims), flags)
            inv = W.inventories()
            tables, nodes = _place(W, w.claims, pod_off, first, co, None, len(w.claims), flags)
            for r in range(3):
                assert tables[r].tobytes() == ref[r].tobytes(), f"flags {flags} rank {r}"
                assert W.inventories()[r].tobytes() == inv[r].tobytes()
    finally:
        W.close()


def test_world1_equals_single_inventory_call(pkg):
    """World 1 over [0, n_node), no export: table, pod_node and inventory byte for byte dra_place_pods_batch's."""
    api = pkg.api
    rng = np.random.default_rng(3)
    w, pod_off = pkg.synth.pods(800, 19, 13)
    n_pod = len(pod_off) - 1
    cn = rng.integers(0, w.n_node + 2, n_pod * 8).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 8).astype(np.uint32)
    W = _world(pkg, w, 1, [0, w.n_node], 0)
    with api.Context(device=0) as single:
        single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
        try:
            for flags in _flags(api):
                for c_, o_ in ((cn, co), (None, None)):
                    tables, nodes = _place(W, w.claims, pod_off, c_, o_, None, len(w.claims), flags)
                    out, pod_node = single.place_pods(w.claims, pod_off, c_, o_, None, len(w.claims), flags)
                    assert tables[0].tobytes() == out.tobytes() and nodes[0].tobytes() == pod_node.tobytes()
                    assert W.ctxs[0].get_inventory().tobytes() == single.get_inventory().tobytes(), f"flags {flags}"
            assert "place_shard" in W.ctxs[0].last_chain() and "pod_gather" not in W.ctxs[0].last_chain()
        finally:
            W.close()


def test_errors(pkg):
    """Host-side refusals return before anything is enqueued.  Each device-detected fault gives DRA_E_INVAL on EVERY rank
    with the live and pristine inventories unchanged, and the next valid call on the same world is right."""
    import torch
    R, api = pkg.records, pkg.api
    w, pod_off = pkg.synth.pods(60, 11, 3)
    n_pod = len(pod_off) - 1
    bounds = [0, 5, 11]
    rng = np.random.default_rng(1)
    cn = rng.integers(0, w.n_node, n_pod * 4).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 4).astype(np.uint32)
    d_c, d_p, d_n, d_o, d_pn = S.dev(w.claims), S.dev(pod_off), S.dev(cn), S.dev(co), S.dev(np.zeros(n_pod, np.uint32))
    torch.cuda.synchronize()

    def raw(c, **k):
        a = dict(claims=d_c.data_ptr(), n_claim=len(w.claims), pod_off=d_p.data_ptr(), n_pod=n_pod, cn=d_n.data_ptr(),
                 co=d_o.data_ptr(), n_pair=len(cn), out_off=None, n_out=len(w.claims), pod_node=d_pn.data_ptr(), flags=0)
        a.update(k)
        return c._lib.dra_place_pods_batch_global_device(c._h, a["claims"], a["n_claim"], a["pod_off"], a["n_pod"], a["cn"],
                                                         a["co"], a["n_pair"], a["out_off"], a["n_out"], a["pod_node"],
                                                         a["flags"])

    with api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        assert raw(c) == api.E_STATE                                         # no shard
        c.comm_init_local(0, 2); c.set_shard(0, 5, take_stray=True)
        assert raw(c) == api.E_STATE                                         # world 2 after a bare set_shard
        c.set_shard_map(bounds, 0)
        assert raw(c) == api.E_STATE                                         # world 2 without export + import
    W = _world(pkg, w, 2, bounds, 1, max_pods=n_pod)
    try:
        c0 = W.ctxs[0]
        with pytest.raises(api.DraError) as e:
            c0.set_shard_place(n_pod)                                        # after the export
        assert e.value.code == api.E_STATE
        assert raw(c0, flags=0x80) == api.E_INVAL                            # unknown flag
        assert raw(c0, flags=api.F_NODE_SORTED) == api.E_INVAL
        assert raw(c0, n_out=N_OUT_MAX + 1) == api.E_INVAL                   # past the exported table
        assert raw(c0, n_out=len(w.claims) - 1) == api.E_INVAL               # n_out < n_claim without out_off
        assert raw(c0, n_pod=0) == api.E_INVAL                               # claims but no pods
        assert raw(c0, cn=None) == api.E_INVAL                               # candidates: both or neither
        assert raw(c0, cn=None, co=None) == api.E_INVAL                      # dense form with n_pair != 0
        assert raw(c0, n_pod=n_pod + 1) == api.E_STATE                       # beyond max_pods of the export
        assert raw(c0, pod_node=None) == api.E_INVAL
        _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), 0, "after host-side refusals")
        bad_po = pod_off.copy(); bad_po[5] = bad_po[7] + 1
        short_po = pod_off.copy(); short_po[-1] -= 1
        bad_co = co.copy(); bad_co[3] = bad_co[5] + 1
        long_co = co.copy(); long_co[-1] += 1                                # cand_off[n_pod] = n_pair + 1
        past = np.arange(len(w.claims), dtype=np.uint32); past[-1] = len(w.claims)
        for what, po, co_, oo, flags in (("pod_off not monotone", bad_po, co, None, 0),
                                         ("pod_off short", short_po, co, None, api.F_FRESH_INVENTORY),
                                         ("cand_off not monotone", pod_off, bad_co, None, api.F_EXHAUSTIVE),
                                         ("cand_off not spanning", pod_off, long_co, None, api.F_FRESH_INVENTORY),
                                         ("slot past n_out", pod_off, co, past, 0)):
            before = W.inventories()
            S.place(W, w.claims, po, (cn, co_), oo, len(w.claims), flags, n_pair=len(cn), expect=api.E_INVAL)
            for b, a in zip(before, W.inventories()):
                assert a.tobytes() == b.tobytes(), f"{what}: a failed call changed an inventory"
            _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), api.F_EXHAUSTIVE, f"after {what}")
        # the pristine copies are untouched: a fresh call answers from the inventory as loaded
        _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), api.F_FRESH_INVENTORY, "fresh after the faults")
    finally:
        W.close()
    # a rank that could finalise more slots than the packet room its export reserved: every rank fails, nothing changes
    W = _world(pkg, w, 2, bounds, 1, cap_per_rank=8)
    try:
        before = W.inventories()
        S.place(W, w.claims, pod_off, (cn, co), None, len(w.claims), 0, expect=api.E_INVAL)
        for b, a in zip(before, W.inventories()):
            assert a.tobytes() == b.tobytes()
        one = np.array([0, int(pod_off[1])], np.uint32)                      # one pod: within the room
        _check(W, w, w.claims[: one[1]], one, cn[:4], co[:2], None, int(one[1]), 0, "within the packet room")
    finally:
        W.close()


def test_import_refuses_a_peer_set_up_differently(pkg):
    """dra_set_shard_place's size is part of the peer buffer's layout."""
    api = pkg.api
    w, _ = pkg.synth.pods(50, 8, 1)
    ctxs = [api.Context(device=0) for _ in range(2)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, 2)
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard_map([0, 4, 8], 0)
            c.set_shard_place(100 + r)
            c.shard_export(1024, 0, want_handle=False)
        with pytest.raises(api.DraError) as e:
            ctxs[0].peer_import_local(ctxs)
        assert e.value.code == api.E_INVAL
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("world", [2, 4])
def test_classic_flow_without_a_sync(pkg, oracle, world):
    """Exhaustive sharded UnsuitableNodes -> sharded place on the suitable nodes -> claims' node fields set from pod_node
    -> sharded Deallocate of the table -> inventory sync: every rank holds the starting inventory again."""
    import torch
    R, api = pkg.records, pkg.api
    w, pod_off = pkg.synth.pods(300, 24, 40 + world)
    n_pod = len(pod_off) - 1
    bounds = S.bounds(w.n_node, world, "even")
    n_pair = n_pod * w.n_node
    W = _world(pkg, w, world, bounds, 0, max_pairs=n_pair)
    try:
        bits = S.unsuitable(W, w.claims, pod_off, flags=api.F_EXHAUSTIVE)
        verdict = np.unpackbits(bits[0], bitorder="little")[:n_pair].reshape(n_pod, w.n_node)
        dn, do = S.dense(n_pod, w.n_node)
        ref_bits = oracle.unsuitable(w.gpus, w.node_off, w.table, w.claims, pod_off, dn, do, flags=oracle.F_EXHAUSTIVE)
        assert np.packbits(verdict.ravel(), bitorder="little").tobytes() == ref_bits.tobytes()
        cn, co = _flat([list(np.flatnonzero(verdict[p])) for p in range(n_pod)])
        ref, ref_node = _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), api.F_EXHAUSTIVE, "place on the verdict")
        assert (ref_node != NONE).sum() > n_pod // 4
        claims = w.claims.copy()
        for p in range(n_pod):
            claims["node"][pod_off[p]: pod_off[p + 1]] = ref_node[p] if ref_node[p] != NONE else 0
        table, d_c2 = S.dev(ref), S.dev(claims)
        torch.cuda.synchronize()
        for c in W.ctxs:                                 # the release and the sync enqueued with no wait in between
            c.deallocate_global_device(d_c2.data_ptr(), len(claims), None, table.data_ptr(), len(claims))
        W.assert_synced(w.gpus, "the release of the placed table")
    finally:
        W.close()
