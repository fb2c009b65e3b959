"""GPU suite: Deallocate on a sharded world (dra_deallocate_batch_global_device).  World contexts of this process on ONE
device, wired like test_gpu_shard_sync.py.  The CPU oracle runs spec §9 on ONE whole inventory.  After each sharded
Deallocate (a) every rank's own GPU range equals the oracle's state byte for byte, (b) every GPU outside a rank's range is
byte for byte what that rank held before the call, and (c) after an inventory sync every rank's whole inventory equals the
oracle's."""
import os

import numpy as np
import pytest

import shard_world as S

pytestmark = pytest.mark.gpu


def _world(pkg, w, world, bounds, stray_rank, max_pairs=None):
    return S.World(pkg, w.table, w.node_off, w.gpus, world, bounds, stray_rank, n_out_max=1 << 16, pairs=max_pairs)


def _pods_allocate(pkg, oracle, W, w, rng, state, flags, oflags):
    pc, po, poo, pn = S.malformed_mixed(pkg, w, W.bounds, rng, True)
    ref, state = oracle.allocate_pods(state, w.node_off, w.table, pc, po, poo, pn, oflags)
    S.same_tables(S.pods(W, pc, po, poo, pn, flags), ref, f"sharded pods Allocate flags {flags}")
    return pc, poo, pn, ref, state


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_mixed_sequence_released_from_gathered_tables(pkg, oracle, world):
    """Sharded Allocate with SHARED claims, then sharded pods Allocate first-fit and exhaustive; each table is released by
    the sharded Deallocate straight from the rank's gathered table.  No rank's copy of any GPU gets a share count at or
    above 0x8000 (the wrap a per-rank dra_deallocate_batch of the gathered records causes), and two kernels per call."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(300 + world)
    w = pkg.synth.mixed(2400, 31, 170 + world, invalid=True)
    kind = {1: "even", 2: "uneven", 3: "empty", 4: "uneven"}[world]
    W = _world(pkg, w, world, S.bounds(w.n_node, world, kind), world - 1)
    try:
        state = w.gpus.copy()
        claims = S.shared_mixed(pkg, w, rng)
        out_off, n_out = R.out_offsets(claims, w.n_node)
        ref, state = oracle.allocate(state, w.node_off, w.table, claims, out_off, int(n_out))
        S.same_tables(S.allocate(W, claims, out_off, int(n_out)), ref, "sharded Allocate")
        shared_ok = (ref["status"] == R.ST_OK) & (ref["profile"] == R.PROFILE_SHARED)
        assert shared_ok.any() and (ref["size"][ref["status"] == R.ST_OK] > 0).any()
        state = oracle.deallocate(state, claims, ref, out_off, n_node=w.n_node)
        S.deallocate(W, claims, out_off, int(n_out), state, "release of the Allocate", ptrs=[S.table_ptr(c) for c in W.ctxs])
        for flags, oflags in ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            pc, poo, pn, ref, state = _pods_allocate(pkg, oracle, W, w, rng, state, flags, oflags)
            assert (ref["status"] == R.ST_OK).any()
            state = oracle.deallocate(state, pc, ref, poo, n_node=w.n_node)
            S.deallocate(W, pc, poo, pn, state, f"release of the pods flags {flags}", ptrs=[S.table_ptr(c) for c in W.ctxs])
        for r, inv in enumerate(W.inventories()):
            assert (inv["share_cnt"] < 0x8000).all(), f"rank {r}: a share count wrapped"
        assert state.tobytes() == w.gpus.tobytes(), "releasing every table must give back the loaded inventory"
        W.assert_synced(state, "after the sequence")
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_release_a_subset_then_allocate_and_unsuitable(pkg, oracle, world):
    """A random subset of a sharded Allocate's claims, with their out_off into the full gathered table, is released.  A
    further sharded Allocate and a sharded UnsuitableNodes (dense and candidate lists, first-fit and exhaustive) then answer
    as the oracle does on the resulting state, and the new Allocate takes GPUs the release freed."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(40 + world)
    w = pkg.synth.mixed(3000, 29, 60 + world, invalid=True)
    n_pod_uns = 200
    W = _world(pkg, w, world, S.bounds(w.n_node, world, "uneven" if world == 3 else "even"), world - 1,
                     max_pairs=n_pod_uns * w.n_node)
    try:
        claims = S.shared_mixed(pkg, w, rng)
        out_off, n_out = R.out_offsets(claims, w.n_node)
        ref, full = oracle.allocate(w.gpus, w.node_off, w.table, claims, out_off, int(n_out))
        S.same_tables(S.allocate(W, claims, out_off, int(n_out)), ref, "sharded Allocate")
        sel = np.sort(rng.choice(len(claims), len(claims) // 3, replace=False))
        sub, sub_off = claims[sel].copy(), out_off[sel].copy()
        state = oracle.deallocate(full, sub, ref, sub_off, n_node=w.n_node)
        assert state.tobytes() != full.tobytes()
        S.deallocate(W, sub, sub_off, int(n_out), state, "subset release", ptrs=[S.table_ptr(c) for c in W.ctxs])
        slots = R.claim_slots(sub, w.n_node)
        freed = {int(ref["gpu"][int(o) + k]) for o, s in zip(sub_off, slots) for k in range(int(s))
                 if ref["status"][int(o) + k] == R.ST_OK}
        c2 = S.shared_mixed(pkg, w, rng)
        o2, n2 = R.out_offsets(c2, w.n_node)
        ref2, state2 = oracle.allocate(state, w.node_off, w.table, c2, o2, int(n2))
        assert ref2.tobytes() != oracle.allocate(full, w.node_off, w.table, c2, o2, int(n2))[0].tobytes()
        S.same_tables(S.allocate(W, c2, o2, int(n2)), ref2, "sharded Allocate after the release")
        assert freed & set(ref2["gpu"][ref2["status"] == R.ST_OK].tolist()), "the freed capacity was not reused"
        uc = c2[:900]
        upo = np.unique(np.concatenate([[0, 900], rng.integers(0, 900, n_pod_uns - 20)])).astype(np.uint32)
        n_pod = len(upo) - 1
        cn, co = S.candidates(rng, n_pod, w.n_node)
        for flags, oflags in ((0, 0), (api.F_EXHAUSTIVE, oracle.F_EXHAUSTIVE)):
            for name, dn, do, on, oo in (("dense", None, None) + S.dense(n_pod, w.n_node), ("candidates", cn, co, cn, co)):
                want = oracle.unsuitable(state2, w.node_off, w.table, uc, upo, on, oo, flags=oflags)
                for r, b in enumerate(S.unsuitable(W, uc, upo, None if dn is None else (dn, do), flags)):
                    assert b.tobytes() == want.tobytes(), f"UnsuitableNodes {name} flags {flags}: rank {r} differs"
        W.assert_ranges(None, state2, "after the further Allocate")
        W.assert_synced(state2, "after the release and the further calls")
    finally:
        W.close()


def test_no_peer_is_waited_for(pkg, oracle):
    """World 3 with only bare dra_set_shard and no export or import: the call works, and each rank's call completes and
    is synced before the next rank calls at all."""
    R = pkg.records
    w = pkg.synth.mixed(2400, 31, 5, invalid=True)
    ref, loaded = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, int(w.n_out))
    want = oracle.deallocate(loaded, w.claims, ref, w.out_off, n_node=w.n_node)
    bounds = [0, 9, 20, 31]
    ctxs = [pkg.api.Context(device=0) for _ in range(3)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, 3)
            c.set_table(w.table); c.set_inventory(loaded, w.node_off)
            c.set_shard(bounds[r], bounds[r + 1], take_stray=r == 0)
        d = [S.dev(w.claims), S.dev(w.out_off), S.dev(ref)]
        import torch
        torch.cuda.synchronize()
        for r, c in enumerate(ctxs):
            c.deallocate_global_device(d[0].data_ptr(), len(w.claims), d[1].data_ptr(), d[2].data_ptr(), int(w.n_out))
            c.sync()
            inv = c.get_inventory()
            g0, g1 = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
            assert inv[g0:g1].tobytes() == want[g0:g1].tobytes(), f"rank {r} own range"
            assert inv[:g0].tobytes() == loaded[:g0].tobytes() and inv[g1:].tobytes() == loaded[g1:].tobytes(), f"rank {r}"
        assert want.tobytes() != loaded.tobytes() and (ref["status"] == R.ST_OK).any()
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("bounds", [[0, 2, 4], [0, 1, 3, 4]])
def test_slots_counted_on_the_whole_inventory(pkg, oracle, bounds):
    """slots(c) is counted on the whole inventory's node indices, whichever rank owns the node: a GPU claim naming another
    rank's node has `count` slots, one naming no node has one.  Here rank 0 releases the records of a count-3 claim on
    the last rank's node, which lie on rank 0's GPUs, and a count-3 claim naming no node owns ONE slot (were it three, its
    range would leave n_out and the call would fail)."""
    R = pkg.records
    gpus, node_off = R.make_inventory([4] * 4, mig=True)
    gpus["flags"] |= R.GPU_FULL_ALLOCATED; gpus["busy"] = 0xFF
    claims = np.zeros(3, dtype=R.CLAIM_DTYPE)
    claims[0] = (R.KIND_GPU, 0, 3, 3, 0, 0)                  # count 3 on node 3: slots 0-2
    claims[1] = (R.KIND_GPU, 0, 3, 99, 0, 0)                 # count 3, no node: slot 3 only
    claims[2] = (R.KIND_MIG, 1, 1, 0, 0, 0)                  # slot 4
    out_off = np.array([0, 3, 4], dtype=np.uint32)
    out = np.zeros(5, dtype=R.OUT_DTYPE)
    out["gpu"] = [0, 1, 2, 13, 3]
    out["start"], out["size"], out["profile"], out["status"] = [0, 0, 0, 0, 2], [0, 0, 0, 0, 2], [0xFF] * 4 + [1], R.ST_OK
    w = type("W", (), {})()
    w.gpus, w.node_off, w.table, w.n_node = gpus, node_off, R.default_table(), 4
    W = _world(pkg, w, len(bounds) - 1, bounds, len(bounds) - 2)
    try:
        want = oracle.deallocate(gpus, claims, out, out_off, n_node=4)
        assert not (want["flags"][[0, 1, 2, 13]] & R.GPU_FULL_ALLOCATED).any() and want["busy"][3] == 0xF3
        S.deallocate(W, claims, out_off, 5, want, f"bounds {bounds}", out=out)
        W.assert_synced(want, f"bounds {bounds}")
    finally:
        W.close()


def _contended(pkg, rng, n_node, per_node, n_claim):
    """An inventory fully taken (every slice busy, FULL_ALLOCATED, share counts high) and n_claim claims whose OK records
    pile onto few GPUs: a quarter of the GPUs take most MIG and SHARED records.  Records need not come from an Allocate:
    the spec §9 updates commute, and the oracle applies the same ones."""
    R = pkg.records
    gpus, node_off = R.make_inventory([per_node] * n_node, mig=True)
    n_gpu = len(gpus)
    gpus["busy"] = 0xFFFF; gpus["flags"] |= R.GPU_FULL_ALLOCATED
    gpus["share_cnt"] = 0x6000; gpus["mem_free_mib"] = 1000
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"] = rng.choice(np.array([R.KIND_GPU, R.KIND_MIG, R.KIND_SHARED], dtype=np.uint8), n_claim, p=[0.2, 0.4, 0.4])
    c["node"] = np.where(rng.random(n_claim) < 0.02, n_node + 3, rng.integers(0, n_node, n_claim)).astype(np.uint32)
    c["count"] = np.where(c["kind"] == R.KIND_GPU, rng.integers(1, 4, n_claim), 1).astype(np.uint16)
    c["profile"] = np.where(c["kind"] == R.KIND_MIG, rng.integers(0, 6, n_claim), 0).astype(np.uint8)
    c["mem_limit_mib"] = np.where(c["kind"] == R.KIND_SHARED, rng.integers(1, 40, n_claim), 0).astype(np.uint32)
    out_off, n_out = R.out_offsets(c, n_node)
    out = np.zeros(int(n_out), dtype=R.OUT_DTYPE)
    hot = rng.random(int(n_out)) < 0.8
    out["gpu"] = np.where(hot, rng.integers(0, max(1, n_gpu // 4), int(n_out)), rng.integers(0, n_gpu + 8, int(n_out)))
    size = rng.choice(np.array([1, 2, 4, 8, 16], dtype=np.uint8), int(n_out))
    out["size"] = size
    out["start"] = (rng.integers(0, 16, int(n_out)) % (17 - size.astype(np.int64))).astype(np.uint8)
    out["status"] = np.where(rng.random(int(n_out)) < 0.9, R.ST_OK, R.ST_NO_CAPACITY).astype(np.uint8)
    return gpus, node_off, c, out_off, int(n_out), out


def test_many_ctas_with_contended_atomics(pkg, oracle):
    """240,000 claims (the apply kernel spans 938 CTAs) over 1,024 GPUs, most MIG and SHARED records on 256 of them."""
    rng = np.random.default_rng(23)
    gpus, node_off, claims, out_off, n_out, out = _contended(pkg, rng, 128, 8, 240_000)
    w = type("W", (), {})()
    w.gpus, w.node_off, w.table, w.n_node = gpus, node_off, pkg.records.default_table(), len(node_off) - 1
    W = _world(pkg, w, 3, [0, 30, 31, 128], 1)
    try:
        state = oracle.deallocate(gpus, claims, out, out_off, n_node=w.n_node)
        S.deallocate(W, claims, out_off, n_out, state, "contended release", out=out)
        W.assert_synced(state, "contended release")
    finally:
        W.close()


def _parity_records(pkg, w, rng, with_off):
    """Claims and records covering every branch of slots(c) and of the apply: multi-count GPU claims, claims naming no
    node, INVALID / POD / SEARCH_LIMIT / NO_CAPACITY records, and OK records whose gpu is n_gpu or beyond."""
    R = pkg.records
    claims = w.claims.copy()
    claims["kind"][:40], claims["count"][:40], claims["node"][:40] = R.KIND_GPU, 3, 2          # count 3 on a node
    claims["node"][40:60] = w.n_node + 1                                                        # naming no node
    claims["kind"][60:70], claims["count"][60:70] = R.KIND_GPU, 0                              # count 0: one slot
    if with_off:
        out_off, n_out = R.out_offsets(claims, w.n_node)
        n_out = int(n_out)
    else:
        out_off, n_out = None, len(claims)
    out = np.zeros(n_out, dtype=R.OUT_DTYPE)
    out["gpu"] = rng.integers(0, w.n_gpu, n_out)
    out["gpu"][::37] = w.n_gpu + rng.integers(0, 5, len(out["gpu"][::37]))
    out["gpu"][::53] = R.GPU_NONE
    out["size"] = rng.choice(np.array([1, 2, 3, 4, 7, 8], dtype=np.uint8), n_out)
    out["start"] = rng.integers(0, 8, n_out)
    out["profile"] = rng.integers(0, 16, n_out)
    st = np.full(n_out, R.ST_OK, dtype=np.uint8)
    pick = rng.random(n_out)
    st[pick < 0.25] = rng.choice(np.array([R.ST_INVALID, R.ST_POD, R.ST_SEARCH_LIMIT, R.ST_NO_CAPACITY], dtype=np.uint8),
                                 int((pick < 0.25).sum()))
    out["status"] = st
    return claims, out_off, n_out, out


@pytest.mark.parametrize("with_off", [True, False])
def test_world1_equals_deallocate_batch(pkg, oracle, with_off):
    """World 1 over [0, n_node): byte for byte what dra_deallocate_batch leaves, on the same inputs and the same start."""
    R = pkg.records
    rng = np.random.default_rng(11 + with_off)
    w = pkg.synth.mixed(2400, 31, 12, invalid=True)
    _, loaded = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, int(w.n_out))
    loaded["share_cnt"] += 200                                 # room for the arbitrary SHARED records below
    claims, out_off, n_out, out = _parity_records(pkg, w, rng, with_off)
    assert (out["status"] == R.ST_OK).sum() > n_out // 2
    w1 = type("W", (), {})()
    w1.gpus, w1.node_off, w1.table, w1.n_node = loaded, w.node_off, w.table, w.n_node
    W = _world(pkg, w1, 1, [0, w.n_node], 0)
    with pkg.api.Context(device=0) as single:
        single.set_table(w.table); single.set_inventory(loaded, w.node_off)
        try:
            want = oracle.deallocate(loaded, claims, out, out_off, n_node=w.n_node)
            S.deallocate(W, claims, out_off, n_out, want, "world 1", out=out)
            single.deallocate(claims, out, out_off)
            assert W.ctxs[0].get_inventory().tobytes() == single.get_inventory().tobytes()
            assert want.tobytes() != loaded.tobytes()
        finally:
            W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_problems_replayed_sharded(pkg, oracle, world):
    """The oracle property generator's problems with random bounds and stray rank: first the records the oracle's Allocate
    produced, then the same records with statuses flipped and GPU indices moved to other ranks' GPUs or past n_gpu."""
    from hypothesis import HealthCheck, given, settings
    from hypothesis import strategies as st
    from test_oracle_properties import problems
    R, api = pkg.records, pkg.api
    n_ex = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))
    big, big_off = R.make_inventory([9] * 4, mig=True)        # the generator's largest inventory: the sync's staging
    ctxs = [api.Context(device=0) for _ in range(world)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, world)
            c.set_inventory(big, big_off)
            c.shard_export(4096, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)

        @settings(max_examples=n_ex or 60, deadline=None, suppress_health_check=list(HealthCheck), derandomize=n_ex == 0,
                  database=None)
        @given(problems(), st.data())
        def run(prob, data):
            g, off, t, c, out_off, n_out = prob
            n_node, n_gpu, n_out = len(off) - 1, len(g), int(n_out)
            cuts = sorted(data.draw(st.lists(st.integers(0, n_node), min_size=world - 1, max_size=world - 1)))
            bounds = [0] + cuts + [n_node]
            stray = data.draw(st.integers(0, world - 1))
            ref, loaded = oracle.allocate(g, off, t, c, out_off, n_out)
            loaded["share_cnt"] += 40
            moved = ref[:n_out].copy()
            for k in range(n_out):
                if data.draw(st.integers(0, 2)) == 0:            # flip: OK <-> INVALID / NO_CAPACITY / POD / SEARCH_LIMIT
                    moved["status"][k] = R.ST_OK if moved["status"][k] else data.draw(st.sampled_from([1, 5, 6, 7]))
                where = data.draw(st.integers(0, 3))
                if where == 1 and n_gpu:                         # any GPU, most often another rank's
                    moved["gpu"][k] = data.draw(st.integers(0, n_gpu - 1))
                elif where == 2:                                 # past the inventory
                    moved["gpu"][k] = n_gpu + data.draw(st.integers(0, 3))
                assert moved["size"][k] <= 16
            w = type("W", (), {})()
            w.gpus, w.node_off, w.table, w.n_node = loaded, off, t, n_node
            W = S.World.__new__(S.World)                 # the contexts above, on this problem's inventory and ranges
            W.pkg, W.table, W.node_off, W.n_node, W.world, W.bounds, W.ctxs, W.loaded = \
                pkg, t, off, n_node, world, bounds, ctxs, [loaded] * world
            for recs, what in ((ref, "the Allocate's records"), (moved, "moved records")):
                for x in ctxs:
                    x.set_table(t); x.set_inventory(loaded, off); x.set_shard_map(bounds, stray_rank=stray)
                if len(c) == 0:
                    continue
                want = oracle.deallocate(loaded, c, recs, out_off, n_node=n_node)
                S.deallocate(W, c, out_off, n_out, want, f"{what}, bounds {bounds}", out=recs[:n_out])
                W.assert_synced(want, f"{what}, bounds {bounds}")

        run()
    finally:
        for c in ctxs:
            c.close()


def test_pinned_host_buffers(pkg, oracle):
    """dra_host_alloc'ed claims, out_off and OutRecs give what device pointers give."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(3)
    w = pkg.synth.mixed(2400, 31, 33, invalid=True)
    ref, loaded = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, int(w.n_out))
    w1 = type("W", (), {})()
    w1.gpus, w1.node_off, w1.table, w1.n_node = loaded, w.node_off, w.table, w.n_node
    sel = np.sort(rng.choice(len(w.claims), 1500, replace=False))
    claims, out_off, n_out = w.claims[sel].copy(), w.out_off[sel].copy(), int(w.n_out)
    want = oracle.deallocate(loaded, claims, ref, out_off, n_node=w.n_node)
    got = []
    for pinned in (True, False):
        W = _world(pkg, w1, 3, [0, 4, 17, 31], 2)
        try:
            if pinned:
                bufs = [api.PinnedBuffer(len(claims), R.CLAIM_DTYPE), api.PinnedBuffer(len(out_off), np.uint32),
                        api.PinnedBuffer(n_out, R.OUT_DTYPE)]
                for b, a in zip(bufs, (claims, out_off, ref[:n_out])):
                    b.array[:] = a
                before, l0 = W.inventories(), [c.launch_count() for c in W.ctxs]
                W.each(lambda r, c: c.deallocate_global_device(bufs[0].ptr, len(claims), bufs[1].ptr, bufs[2].ptr, n_out))
                assert all(c.launch_count() == l + 2 for c, l in zip(W.ctxs, l0))
                W.assert_ranges(before, want, "pinned buffers")
                for b in bufs:
                    b.free()
            else:
                S.deallocate(W, claims, out_off, n_out, want, "device pointers", out=ref[:n_out])
            got.append(W.inventories())
            W.assert_synced(want, "pinned" if pinned else "device")
        finally:
            W.close()
    for a, b in zip(*got):
        assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("world", [1, 3])
def test_bad_slot_range_changes_nothing(pkg, oracle, world):
    """One claim's slots leave n_out, first or last in the array: DRA_E_INVAL at sync on every rank, every live inventory
    byte for byte as before.  The next call on each context succeeds, and a DRA_F_FRESH_INVENTORY sharded Allocate still
    starts from the loaded inventory."""
    R, api = pkg.records, pkg.api
    rng = np.random.default_rng(8 + world)
    w = pkg.synth.mixed(2400, 31, 44, invalid=True)
    W = _world(pkg, w, world, S.bounds(w.n_node, world, "uneven"), 0)
    try:
        claims = S.shared_mixed(pkg, w, rng)
        claims["kind"][-1], claims["count"][-1], claims["node"][-1] = R.KIND_GPU, 2, 3
        out_off, n_out = R.out_offsets(claims, w.n_node)
        n_out = int(n_out)
        ref, state = oracle.allocate(w.gpus, w.node_off, w.table, claims, out_off, n_out)
        S.same_tables(S.allocate(W, claims, out_off, n_out), ref, "sharded Allocate")
        first, last = out_off.copy(), out_off.copy()
        first[0] = n_out                                       # one slot at n_out
        last[-1] = n_out - 1                                   # two slots from n_out - 1
        for bad, what in ((first, "first"), (last, "last")):
            before = W.inventories()
            S.deallocate(W, claims, bad, n_out, out=ref, expect=api.E_INVAL)
            for r, (b, a) in enumerate(zip(before, W.inventories())):
                assert a.tobytes() == b.tobytes(), f"bad slot range {what}: rank {r} inventory changed"
        state = oracle.deallocate(state, claims, ref, out_off, n_node=w.n_node)
        S.deallocate(W, claims, out_off, n_out, state, "after the refused calls", out=ref)
        c2 = S.shared_mixed(pkg, w, rng)
        o2, n2 = R.out_offsets(c2, w.n_node)
        ref2, state2 = oracle.allocate(w.gpus, w.node_off, w.table, c2, o2, int(n2))
        S.same_tables(S.allocate(W, c2, o2, int(n2), api.F_FRESH_INVENTORY), ref2, "fresh Allocate")
        W.assert_ranges(None, state2, "fresh Allocate")
    finally:
        W.close()


def test_refusals_and_empty_calls(pkg):
    """Each refusal returns before anything is enqueued (launch_count unchanged, inventory unchanged); so does n_claim 0."""
    import torch
    R, api = pkg.records, pkg.api
    w = pkg.synth.mixed(600, 11, 3, invalid=True)
    small = pkg.synth.mixed(200, 5, 4, invalid=True)
    d_c, d_o, d_r = S.dev(w.claims), S.dev(w.out_off), S.dev(np.zeros(int(w.n_out), dtype=R.OUT_DTYPE))
    torch.cuda.synchronize()

    def raw(c, **k):
        a = dict(claims=d_c.data_ptr(), n_claim=len(w.claims), out_off=d_o.data_ptr(), out=d_r.data_ptr(), n_out=int(w.n_out))
        a.update(k)
        return c._lib.dra_deallocate_batch_global_device(c._h, a["claims"], a["n_claim"], a["out_off"], a["out"], a["n_out"])

    def refused(c, code, **k):
        inv, n = (c.get_inventory() if c.n_gpu else None), c.launch_count()
        assert raw(c, **k) == code, k
        assert c.launch_count() == n, k
        if inv is not None:
            assert c.get_inventory().tobytes() == inv.tobytes()

    with api.Context(device=0) as c:
        refused(c, api.E_STATE)                                              # no inventory
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        refused(c, api.E_STATE)                                              # no shard
        c.comm_init_local(1, 2); c.set_shard(5, 11)
        refused(c, api.E_INVAL, claims=None)
        refused(c, api.E_INVAL, out=None)
        refused(c, api.E_INVAL, out_off=None, n_out=len(w.claims) - 1)      # n_out < n_claim without out_off
        refused(c, api.E_INVAL, n_claim=(1 << 26) + 1)
        refused(c, api.E_INVAL, n_out=(1 << 26) + 1)
        refused(c, api.OK, n_claim=0)                                        # empty: nothing enqueued
        refused(c, api.OK, n_claim=0, claims=None, out=None, out_off=None, n_out=0)
        c.set_inventory(small.gpus, small.node_off)                          # the shard [5, 11) is past the 5 nodes
        refused(c, api.E_STATE)
        c.set_shard(0, 5, take_stray=True)
        n = c.launch_count()
        assert raw(c, n_claim=0) == api.OK and c.launch_count() == n
        c.sync()
