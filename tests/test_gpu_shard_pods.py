"""GPU suite: pods Allocate on a sharded world (dra_allocate_pods_batch_global_device).  World contexts of this process on
ONE device, wired with dra_comm_init_local / dra_peer_import_local like test_gpu_shard_unsuitable.py.  Every rank's whole
table must be byte for byte the oracle's answer on the world's real state (the inventory each rank holds for its own node
range), each rank's own GPU range the oracle's inventory afterwards, and no rank may write GPUs outside its range."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

import shard_world as S

pytestmark = pytest.mark.gpu

N_OUT_MAX = 1 << 16


def _world(pkg, w, world, bounds, stray_rank=0, max_pairs=None, attrs=None, sels=None, cap_per_rank=0):
    """every rank holding the whole inventory"""
    return S.World(pkg, w.table, w.node_off, w.gpus, world, bounds, stray_rank, attrs, sels, n_out_max=N_OUT_MAX,
                   cap_per_rank=cap_per_rank, pairs=max_pairs)


def _check(W, oracle, w, claims, pod_off, out_off, n_out, flags, what):
    """One call against the oracle on the world's state (the pristine inventory under F_FRESH_INVENTORY): every rank's
    whole table, its own range the oracle's, nothing written outside it."""
    api = W.pkg.api
    before = W.inventories()
    src = w.gpus if flags & api.F_FRESH_INVENTORY else W.state()
    oflags = oracle.F_EXHAUSTIVE if flags & api.F_EXHAUSTIVE else 0
    ref, ref_inv = oracle.allocate_pods(src, w.node_off, w.table, claims, pod_off, out_off, n_out, oflags)
    S.same_tables(S.pods(W, claims, pod_off, out_off, n_out, flags), ref, what)
    W.assert_ranges(before, ref_inv, what)
    return ref


def _flags(api):
    return [0, api.F_EXHAUSTIVE, api.F_FRESH_INVENTORY, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY]


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("workload", ["pods", "mixed_off", "mixed_nooff"])
def test_matches_oracle(pkg, oracle, world, workload):
    """Every flag combination, one after the other on the same world; every rank's whole table and own range checked."""
    api = pkg.api
    rng = np.random.default_rng(world * 7 + len(workload))
    kind = ["even", "uneven", "empty", "even"][world - 1] if world > 1 else "even"
    stray = world - 1                                    # stray_rank != 0 from world 2 on
    attrs = sels = None
    if workload == "pods":
        w, pod_off = pkg.synth.pods(700, 29, world)
        bounds = S.bounds(w.n_node, world, kind)
        jobs = [(w.claims, pod_off, None, w.n_claim)]
    else:
        w = pkg.synth.mixed(2400, 31, 60 + world, invalid=True)
        attrs, sels = pkg.synth.with_selectors(w, world)
        bounds = S.bounds(w.n_node, world, kind)
        jobs = [S.malformed_mixed(pkg, w, bounds, rng, workload == "mixed_off")]
    W = _world(pkg, w, world, bounds, stray, attrs=attrs, sels=sels)
    oracle.set_selectors(attrs, sels)
    try:
        for flags in _flags(api):
            for claims, po, oo, n_out in jobs:
                ref = _check(W, oracle, w, claims, po, oo, n_out, flags, f"{workload} flags {flags}")
                st = ref["status"]
                if flags in (0, api.F_FRESH_INVENTORY):
                    assert (st == pkg.records.ST_OK).any() and (st == pkg.records.ST_POD).any()
                if workload != "pods":
                    assert (st == pkg.records.ST_INVALID).any()
        if workload == "pods":
            ff = oracle.allocate_pods(w.gpus, w.node_off, w.table, w.claims, pod_off)[0]
            ex = oracle.allocate_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, flags=oracle.F_EXHAUSTIVE)[0]
            assert ff.tobytes() != ex.tobytes(), "the workload does not separate first-fit from the exhaustive search"
    finally:
        oracle.set_selectors()
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_allocate_then_pods(pkg, oracle, world):
    """The gap the call closes: after a sharded Allocate without F_FRESH_INVENTORY each rank's copy is right for its own
    nodes only.  dra_allocate_pods_batch on rank 0 answers from its stale copy; the sharded call answers on the real state."""
    R = pkg.records
    w, pod_off = pkg.synth.pods(900, 32, 40 + world)
    bounds = S.bounds(w.n_node, world, "even")
    W = _world(pkg, w, world, bounds, 0)
    try:
        half = int(pod_off[450])
        S.allocate(W, w.claims[:half], None, half)
        real = W.state()
        _, ref_real = oracle.allocate(w.gpus, w.node_off, w.table, w.claims[:half])
        assert real.tobytes() == ref_real.tobytes()
        claims, po = w.claims[half:], (pod_off[450:] - half).astype(np.uint32)
        ref = oracle.allocate_pods(real, w.node_off, w.table, claims, po, flags=oracle.F_EXHAUSTIVE)[0]
        stale = W.ctxs[0].allocate_pods(claims, po, flags=pkg.api.F_EXHAUSTIVE)
        assert stale.tobytes() != ref.tobytes(), "the workload does not expose the stale copies"
        _check(W, oracle, w, claims, po, None, len(claims), pkg.api.F_EXHAUSTIVE, "after a sharded allocate")
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 4])
def test_world_acts_on_its_own_verdict(pkg, oracle, world):
    """Sharded Allocate -> sharded exhaustive UnsuitableNodes -> for each pod a suitable node (one pod per node), claims
    retargeted there -> the sharded pods Allocate with F_EXHAUSTIVE places every one of those pods."""
    import torch
    R, api = pkg.records, pkg.api
    w, pod_off = pkg.synth.pods(500, 40, 70 + world)
    bounds = S.bounds(w.n_node, world, "uneven")
    first = int(pod_off[200])
    n_pod = 300
    W = _world(pkg, w, world, bounds, world - 1, max_pairs=n_pod * w.n_node)
    try:
        S.allocate(W, w.claims[:first], None, first)
        claims = w.claims[first:].copy()
        po = (pod_off[200:] - first).astype(np.uint32)
        n_pair = n_pod * w.n_node
        verdict = [np.unpackbits(b, bitorder="little")[:n_pair].reshape(n_pod, w.n_node)
                   for b in S.unsuitable(W, claims, po, flags=api.F_EXHAUSTIVE)]
        for v in verdict[1:]:
            assert (v == verdict[0]).all()
        real = W.state()
        dn, do = S.dense(n_pod, w.n_node)
        ref_bits = oracle.unsuitable(real, w.node_off, w.table, claims, po, dn, do, flags=oracle.F_EXHAUSTIVE)
        assert np.packbits(verdict[0].ravel(), bitorder="little").tobytes() == ref_bits.tobytes()
        taken, keep = set(), []
        for p in range(n_pod):
            free = [n for n in np.flatnonzero(verdict[0][p]) if n not in taken]
            if free:
                n = int(free[len(free) // 2]); taken.add(n)
                keep.append((p, n))
        assert len(keep) >= 10
        sel = np.concatenate([np.arange(po[p], po[p + 1]) for p, _ in keep])
        sub = claims[sel].copy()
        sub_off = np.zeros(len(keep) + 1, dtype=np.uint32)
        sub_off[1:] = np.cumsum([po[p + 1] - po[p] for p, _ in keep])
        for k, (_, n) in enumerate(keep):
            sub["node"][sub_off[k]: sub_off[k + 1]] = n
        ref = _check(W, oracle, w, sub, sub_off, None, len(sub), api.F_EXHAUSTIVE, "pods on their suitable nodes")
        assert (ref["status"] == 0).all(), "a pod the exhaustive verdict called suitable was not placed"
    finally:
        W.close()


def test_world1_equals_single_inventory_call(pkg, oracle):
    """World 1 over [0, n_node): OutRecs and inventory byte for byte those of dra_allocate_pods_batch, every flag."""
    R, api = pkg.records, pkg.api
    w = pkg.synth.mixed(2000, 29, 88, invalid=True)
    claims, pod_off, out_off, n_out = S.malformed_mixed(pkg, w, [0, w.n_node], np.random.default_rng(9), True)
    W = _world(pkg, w, 1, [0, w.n_node], 0)
    with api.Context(device=0) as single:
        single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
        try:
            for flags in _flags(api):
                got = S.pods(W, claims, pod_off, out_off, n_out, flags)[0]
                ref = single.allocate_pods(claims, pod_off, out_off, n_out, flags)
                assert got.tobytes() == ref.tobytes(), f"flags {flags}"
                assert W.ctxs[0].get_inventory().tobytes() == single.get_inventory().tobytes(), f"flags {flags}"
            assert W.ctxs[0].last_chain() >= {"pod_shard"} and "pod_gather" not in W.ctxs[0].last_chain()
        finally:
            W.close()


def test_consecutive_calls_interleaved(pkg, oracle):
    """Pods calls of changing size between sharded Allocates and sharded UnsuitableNodes on the same export: the epoch
    parity, the packet cursors and the peer buffer shared by the three calls."""
    import torch
    R, api = pkg.records, pkg.api
    world = 3
    w, pod_off = pkg.synth.pods(3000, 30, 5)
    bounds = S.bounds(w.n_node, world, "uneven")
    W = _world(pkg, w, world, bounds, 1, max_pairs=400 * w.n_node)
    rng = np.random.default_rng(4)
    try:
        for step, n_pod in enumerate([400, 1, 37, 211, 3, 150, 64]):
            if step % 2 == 0:                            # a sharded allocate of a slice of the claims
                lo = int(pod_off[step * 200])
                part = w.claims[lo: lo + 300]
                S.allocate(W, part, None, len(part))
            p0 = int(rng.integers(0, 3000 - n_pod))
            claims = w.claims[pod_off[p0]: pod_off[p0 + n_pod]]
            po = (pod_off[p0: p0 + n_pod + 1] - pod_off[p0]).astype(np.uint32)
            if step % 3 == 1:                            # a sharded exhaustive UnsuitableNodes in between
                bits = S.unsuitable(W, claims, po, flags=api.F_EXHAUSTIVE)
                dn, do = S.dense(n_pod, w.n_node)
                ref = oracle.unsuitable(W.state(), w.node_off, w.table, claims, po, dn, do, flags=oracle.F_EXHAUSTIVE)
                for r, b in enumerate(bits):
                    assert b.tobytes() == ref.tobytes(), f"step {step} rank {r} bits"
            flags = api.F_EXHAUSTIVE if step % 2 else 0
            _check(W, oracle, w, claims, po, None, len(claims), flags, f"step {step}")
        assert W.ctxs[0].last_chain() >= {"pod_shard", "pod_gather"}
    finally:
        W.close()


def test_errors(pkg, oracle):
    """Host-side checks return before anything is enqueued.  Device-side faults (pod_off not monotone or short, slots past
    n_out, a rank owning more slots than its packet room) give DRA_E_INVAL on EVERY rank with no inventory changed, and the
    next valid call is right."""
    import torch
    R, api = pkg.records, pkg.api
    w = pkg.synth.mixed(600, 11, 3, invalid=True)
    bounds = [0, 5, 11]
    pod_off = np.arange(0, 61, 3, dtype=np.uint32)
    claims = w.claims[: pod_off[-1]].copy()
    for p in range(20):
        claims["node"][pod_off[p]: pod_off[p + 1]] = claims["node"][pod_off[p]]
    out_off, n_out = R.out_offsets(claims, w.n_node)
    n_out = int(n_out)
    d_c, d_p, d_o = S.dev(claims), S.dev(pod_off), S.dev(out_off)
    torch.cuda.synchronize()

    def raw(c, **k):
        a = dict(claims=d_c.data_ptr(), n_claim=len(claims), pod_off=d_p.data_ptr(), n_pod=20, out_off=d_o.data_ptr(),
                 n_out=n_out, flags=0)
        a.update(k)
        return c._lib.dra_allocate_pods_batch_global_device(c._h, a["claims"], a["n_claim"], a["pod_off"], a["n_pod"],
                                                            a["out_off"], a["n_out"], a["flags"])

    with api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        assert raw(c) == api.E_STATE                                         # no shard
        c.comm_init_local(0, 2); c.set_shard(0, 5, take_stray=True)
        assert raw(c) == api.E_STATE                                         # world 2 after a bare set_shard
        c.set_shard_map(bounds, 0)
        assert raw(c) == api.E_STATE                                         # world 2 without export + import
    W = _world(pkg, w, 2, bounds, 1)
    try:
        c0 = W.ctxs[0]
        assert raw(c0, flags=0x80) == api.E_INVAL                            # unknown flag
        assert raw(c0, flags=api.F_NODE_SORTED) == api.E_INVAL
        assert raw(c0, n_out=N_OUT_MAX + 1) == api.E_INVAL                   # past the exported table
        assert raw(c0, out_off=None, n_out=len(claims) - 1) == api.E_INVAL   # n_out < n_claim without out_off
        assert raw(c0, n_pod=0) == api.E_INVAL                               # claims but no pods
        assert raw(c0, n_claim=(1 << 26) + 1) == api.E_INVAL
        _check(W, oracle, w, claims, pod_off, out_off, n_out, 0, "after host-side errors")
        bad_po = pod_off.copy(); bad_po[5] = bad_po[7] + 1
        short_po = pod_off.copy(); short_po[-1] -= 1
        past = out_off.copy(); past[-1] = n_out
        for po, oo, flags in ((bad_po, out_off, 0), (short_po, out_off, api.F_FRESH_INVENTORY), (pod_off, past, api.F_EXHAUSTIVE)):
            before = W.inventories()
            S.pods(W, claims, po, oo, n_out, flags, expect=api.E_INVAL)
            for b, a in zip(before, W.inventories()):
                assert a.tobytes() == b.tobytes(), "a failed call changed an inventory"
            _check(W, oracle, w, claims, pod_off, out_off, n_out, api.F_EXHAUSTIVE, "after a device-side error")
    finally:
        W.close()
    # more slots on one rank than the packet room its export reserved: every rank fails, nothing changes
    W = _world(pkg, w, 2, bounds, 1, cap_per_rank=8)
    try:
        before = W.inventories()
        S.pods(W, claims, pod_off, out_off, n_out, 0, expect=api.E_INVAL)
        for b, a in zip(before, W.inventories()):
            assert a.tobytes() == b.tobytes()
        # two pods without out_off (one slot per claim): within the room
        _check(W, oracle, w, claims[:6], pod_off[:3], None, 6, 0, "within the packet room")
    finally:
        W.close()


def test_empty_and_zero_shapes(pkg, oracle):
    """Only empty pods, n_pod == 0, one pod of one claim on the last node, and a world with an empty range."""
    w = pkg.synth.mixed(400, 13, 12, invalid=True)
    world = 4
    W = _world(pkg, w, world, S.bounds(w.n_node, world, "empty"), 2)
    try:
        z = S.dev(np.zeros(4, dtype=np.uint32))
        W.each(lambda r, c: c.allocate_pods_global_device(0, 0, z.data_ptr(), 0, None, 0, 0))
        one = w.claims[:1].copy(); one["node"] = w.n_node - 1
        _check(W, oracle, w, one, np.array([0, 1], dtype=np.uint32), None, 1, 0, "one pod")
        _check(W, oracle, w, w.claims[:0], np.zeros(4, dtype=np.uint32), None, 1, 0, "only empty pods")
        po = np.array([0, 0, 5, 5, 9, 9], dtype=np.uint32)
        c = w.claims[:9].copy(); c["node"][:5] = 0; c["node"][5:] = w.n_node - 1
        _check(W, oracle, w, c, po, None, 9, pkg.api.F_EXHAUSTIVE, "empty pods between")
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_pod_problems_replayed_sharded(pkg, oracle, world):
    """The pod-mode property generator through the sharded call with random bounds and stray rank."""
    from hypothesis import HealthCheck, given, settings
    from hypothesis import strategies as st
    from test_pod_mode import pod_problems
    R, api = pkg.records, pkg.api
    n_ex = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))
    ctxs = [api.Context(device=0) for _ in range(world)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, world)
            c.shard_export(4096, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)

        @settings(max_examples=n_ex or 80, deadline=None, suppress_health_check=list(HealthCheck), derandomize=n_ex == 0,
                  database=None)
        @given(pod_problems(), st.booleans(), st.booleans(), st.data())
        def run(prob, exhaustive, fresh, data):
            g, off, t, c, pod_off, out_off, n_out = prob
            n_node = len(off) - 1
            cuts = sorted(data.draw(st.lists(st.integers(0, n_node), min_size=world - 1, max_size=world - 1)))
            bounds = [0] + cuts + [n_node]
            stray = data.draw(st.integers(0, world - 1))
            for x in ctxs:
                x.set_table(t); x.set_inventory(g, off); x.set_shard_map(bounds, stray_rank=stray)
            w = SimpleNamespace(gpus=g, node_off=off, table=t)
            W = S.World.__new__(S.World)                 # the contexts above, on this problem's inventory and ranges
            W.pkg, W.table, W.node_off, W.n_node, W.world, W.bounds, W.ctxs, W.loaded = \
                pkg, t, off, n_node, world, bounds, ctxs, [g] * world
            flags = (api.F_EXHAUSTIVE if exhaustive else 0) | (api.F_FRESH_INVENTORY if fresh else 0)
            n_out = max(int(n_out), 1)
            if len(pod_off) - 1 == 0:
                return
            _check(W, oracle, w, c, pod_off, out_off, n_out, flags, f"bounds {bounds} stray {stray}")

        run()
    finally:
        for c in ctxs:
            c.close()
