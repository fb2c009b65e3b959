"""GPU suite: the multi-rank paths on ONE device — world contexts of this process, each with its own stream, wired
together with dra_comm_init_local / dra_peer_import_local (the form a single driver process uses; torchrun ranks use
IPC handles instead: tests/multi_gpu_check.py, wrapped by test_gpu_multi_rank.py).  Covers the sharded GLOBAL batch
(device-side range filter, results at global slots, packet all-gather) and the per-rank-slice gather, on the fused and
the sort path, bit-exact with the oracle on the global batch."""
import numpy as np
import pytest

import shard_world as S

pytestmark = pytest.mark.gpu


def _make_world(pkg, world, flags=0):
    ctxs = [pkg.api.Context(device=0, flags=flags) for _ in range(world)]
    for r, c in enumerate(ctxs):
        c.comm_init_local(r, world)
    return ctxs


@pytest.mark.parametrize("world,cfg_flags,seed", [(2, 0, 0), (4, 0, 1), (3, "nofused", 2), (2, 0, 3)])
def test_sharded_global_batch(pkg, oracle, world, cfg_flags, seed):
    R = pkg.records
    flags = pkg.api.CFG_NO_FUSED if cfg_flags == "nofused" else 0
    w = pkg.synth.mixed(6000, 30, 60 + seed, invalid=seed != 3) if seed != 1 else pkg.synth.cfg2(8000, 40)
    out_off = w.out_off
    ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)          # one-time setup, like the inventory
    ctxs = _make_world(pkg, world, flags)
    try:
        for r, c in enumerate(ctxs):
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
            if seed == 3:
                c.set_shard(ranges[r][0], ranges[r][1], take_stray=(r == 0))      # without the map: counts travel in a header
            else:
                c.set_shard_map([x[0] for x in ranges] + [ranges[-1][1]], stray_rank=0)
            c.shard_export(w.n_out, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)
        d_claims = S.dev(w.claims)
        d_off = None if out_off is None else S.dev(out_off)
        ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, out_off, w.n_out)
        for rep in range(4):                                             # repeated calls: parity double-buffering, plan from the hint
            for c in ctxs:                                               # enqueue on every rank, THEN wait
                c.allocate_global_device(d_claims.data_ptr(), w.n_claim, None if d_off is None else d_off.data_ptr(), w.n_out,
                                         pkg.api.F_FRESH_INVENTORY)
            for r, c in enumerate(ctxs):
                got = c.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE))
                assert got.tobytes() == ref.tobytes(), f"rank {r} rep {rep}: table differs from the oracle"
                g0, g1 = int(w.node_off[ranges[r][0]]), int(w.node_off[ranges[r][1]])
                assert c.get_inventory()[g0:g1].tobytes() == ref_inv[g0:g1].tobytes(), f"rank {r}: shard inventory differs"
    finally:
        for c in ctxs:
            c.close()


def test_sharded_global_batch_world1_and_empty_shards(pkg, oracle):
    """world 1 needs no export; a rank whose node range gets no claim; a rank with an empty node range."""
    R = pkg.records
    w = pkg.synth.cfg2(3000, 12)
    w.claims["node"] = w.claims["node"] % 5                              # nodes 5..11 get nothing
    ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard(0, w.n_node, True)
        d = S.dev(w.claims)
        c.allocate_global_device(d.data_ptr(), w.n_claim, None, w.n_out, pkg.api.F_FRESH_INVENTORY)
        assert c.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE)).tobytes() == ref.tobytes()
    ctxs = _make_world(pkg, 3)
    try:
        rng = [(0, 5), (5, 12), (12, 12)]
        for r, c in enumerate(ctxs):
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard_map([0, 5, 12, 12], stray_rank=2)
            c.shard_export(w.n_out, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)
        d = S.dev(w.claims)
        for _ in range(3):
            for c in ctxs:
                c.allocate_global_device(d.data_ptr(), w.n_claim, None, w.n_out, pkg.api.F_FRESH_INVENTORY)
            for c in ctxs:
                assert c.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE)).tobytes() == ref.tobytes()
        # the distribution shifts under a plan made for the old one: every claim now lands in rank 1's range.  The call
        # fails WITHOUT touching anything ("call again"), the peers are told at once (no time-out), the retry succeeds.
        w2 = pkg.synth.cfg2(3000, 12); w2.claims["node"] = 5 + w2.claims["node"] % 7
        ref2, _ = oracle.allocate(w2.gpus, w2.node_off, w2.table, w2.claims)
        d2 = S.dev(w2.claims)
        for c in ctxs:
            c.allocate_global_device(d2.data_ptr(), w2.n_claim, None, w2.n_out, pkg.api.F_FRESH_INVENTORY)
        errs = []
        for c in ctxs:
            try:
                c.gather_read(np.zeros(w2.n_out, dtype=R.OUT_DTYPE))
            except pkg.api.DraError as e:
                errs.append(e.code)
        assert pkg.api.E_STATE in errs, errs
        for c in ctxs:
            c.allocate_global_device(d2.data_ptr(), w2.n_claim, None, w2.n_out, pkg.api.F_FRESH_INVENTORY)
        for c in ctxs:
            assert c.gather_read(np.zeros(w2.n_out, dtype=R.OUT_DTYPE)).tobytes() == ref2.tobytes()
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("world,nofused", [(2, False), (3, True)])
def test_per_rank_slices_gather(pkg, oracle, world, nofused):
    """dra_allocate_batch_gather_device: every rank owns its nodes' inventory and claims; slices + zeroed padding."""
    R = pkg.records
    w = pkg.synth.mixed(5000, 28, 77)
    ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
    lbs = [pkg.shard.local_batch(w.gpus, w.node_off, w.claims, r, ranges) for r in range(world)]
    n_per = max(b.n_out for b in lbs) + 3
    ctxs = _make_world(pkg, world, pkg.api.CFG_NO_FUSED if nofused else 0)
    try:
        for c, lb in zip(ctxs, lbs):
            c.set_table(w.table); c.set_inventory(lb.gpus, lb.node_off)
            c._check(c._lib.dra_peer_export(c._h, n_per, (__import__("ctypes").c_uint8 * 64)()))
        for c in ctxs:
            c.peer_import_local(ctxs)
        dc = [S.dev(lb.claims) for lb in lbs]
        do = [S.dev(lb.out_off) for lb in lbs]
        ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
        for rep in range(3):
            for c, lb, a, b in zip(ctxs, lbs, dc, do):
                c.allocate_gather_device(a.data_ptr(), len(lb.claims), b.data_ptr(), None, lb.n_out, n_per, pkg.api.F_FRESH_INVENTORY)
            for c in ctxs:
                table = c.gather_read(np.zeros(world * n_per, dtype=R.OUT_DTYPE))
                parts = [(b.sel, b.out_off, table[r * n_per: r * n_per + b.n_out], b.gpu_base) for r, b in enumerate(lbs)]
                merged = pkg.shard.merge(w.n_out, w.out_off, parts)
                assert merged.tobytes() == ref.tobytes()
                for r, b in enumerate(lbs):                              # padding of every slice is zero (header promise)
                    assert not table[r * n_per + b.n_out: (r + 1) * n_per].view(np.uint64).any()
    finally:
        for c in ctxs:
            c.close()


def test_device_rendezvous_of_world_contexts(pkg):
    """dra_peer_rendezvous_device: every rank enqueues it, nobody waits on the host in between; repeated calls use
    increasing sequence numbers (nothing to reset); world 1 is a no-op."""
    import torch
    w = pkg.synth.cfg2(2000, 8)
    ctxs = _make_world(pkg, 3)
    try:
        for c in ctxs:
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard_map([0, 3, 6, 8], stray_rank=0)
            c.shard_export(w.n_out, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)
        for _ in range(5):
            l0 = ctxs[1].launch_count()
            for c in ctxs:
                c.peer_rendezvous()
            assert ctxs[1].launch_count() == l0       # (no part of a batch: not counted)
        for c in ctxs:
            c.sync()
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            c.close()
    with pkg.api.Context(device=0) as c:
        c.peer_rendezvous()                      # world 1: nothing to do


# ---- the compaction on one device: world-1 contexts with sub-range shards (no peers, no gather) ---------------------------
# A world-1 context serves [lo, hi) of the inventory and drops every other claim, so each compaction form is checked where
# it matters: the kept claims' positions among dropped ones.  The shard writes the OutRecs of its kept claims only; those
# slots, and the shard's slice of the inventory, must be the oracle's answer to the whole batch (nodes are independent).

@pytest.mark.parametrize("n_claim,compaction", [(262_144, "compact_flat1"), (262_145, "compact_flat8"),
                                                (2_097_152, "compact_flat8"), (2_097_153, "compact_lookback")])
def test_shard_compaction_forms_drop_claims(pkg, oracle, n_claim, compaction):
    """256-claim tiles up to 262,144 claims, 2048-claim tiles up to 2,097,152, the look-back form beyond; strays kept."""
    w = pkg.synth.mixed(n_claim, 2_000, 50, invalid=True)
    ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out, threads=8)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard(500, 1_300, take_stray=True)
        d, o = S.dev(w.claims), S.dev(w.out_off)
        _, _, chain = S.shard_call(pkg, c, w, d, o, 500, 1_300, True, ref, ref_inv, f"{n_claim} claims")
        assert compaction in chain, chain
        outside = np.ones(w.n_gpu, dtype=bool); outside[int(w.node_off[500]):int(w.node_off[1_300])] = False
        assert c.get_inventory()[outside].tobytes() == w.gpus[outside].tobytes(), "a GPU outside the shard changed"


def test_three_shards_cover_the_inventory(pkg, oracle):
    """Three sub-ranges whose union is the whole inventory, strays to the middle one: together they are the oracle's batch."""
    R = pkg.records
    w = pkg.synth.mixed(300_000, 1_500, 51, invalid=True)
    ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out, threads=8)
    merged = np.zeros(w.n_out, dtype=R.OUT_DTYPE)
    covered = np.zeros(w.n_out, dtype=bool)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        d, o = S.dev(w.claims), S.dev(w.out_off)
        for lo, hi, stray in ((0, 400, False), (400, 1_111, True), (1_111, 1_500, False)):
            c.set_shard(lo, hi, take_stray=stray)
            got, m, chain = S.shard_call(pkg, c, w, d, o, lo, hi, stray, ref, ref_inv, f"shard [{lo}, {hi})")
            assert "compact_flat8" in chain, chain
            assert not (covered & m).any()
            merged[m] = got[m]; covered |= m
        assert covered.all() and merged.tobytes() == ref.tobytes()
        assert c.get_inventory().tobytes() == ref_inv.tobytes()


def test_plan_hint_takes_the_staged_kernel_on_a_narrow_shard(pkg, oracle):
    """The first call of a batch size plans for the whole batch (sort path); the second plans from the first call's count
    and, the shard being narrow, lays the staged single-launch kernel out for a few thousand claims."""
    w = pkg.synth.mixed(262_145, 2_000, 52, invalid=True)
    ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out, threads=8)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard(960, 1_000, take_stray=False)
        d, o = S.dev(w.claims), S.dev(w.out_off)
        _, _, first = S.shard_call(pkg, c, w, d, o, 960, 1_000, False, ref, ref_inv, "first call")
        assert "compact_flat8" in first and not first & {"fused_staged", "fused_stream"}, first
        for rep in range(2):
            _, _, chain = S.shard_call(pkg, c, w, d, o, 960, 1_000, False, ref, ref_inv, f"planned call {rep}")
            assert chain == {"compact_flat8", "fused_staged"}, chain


def test_shard_beyond_the_cta_wide_histogram_is_an_error(pkg, oracle):
    """A shard of 12,799 local nodes past the single-launch kernel's limits needs the one-warp histogram, which the sharded
    call does not support: DRA_E_INVAL with the inventory unchanged; one node fewer works."""
    w = pkg.synth.mixed(10_000, 13_000, 53, invalid=True)
    ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off); c.set_shard(0, 12_799, take_stray=True)
        d, o = S.dev(w.claims), S.dev(w.out_off)
        with pytest.raises(pkg.api.DraError) as e:
            c.allocate_global_device(d.data_ptr(), w.n_claim, o.data_ptr(), w.n_out, pkg.api.F_FRESH_INVENTORY)
        assert e.value.code == pkg.api.E_INVAL
        assert c.get_inventory().tobytes() == w.gpus.tobytes()
        c.set_shard(0, 12_798, take_stray=True)
        _, _, chain = S.shard_call(pkg, c, w, d, o, 0, 12_798, True, ref, ref_inv, "12,798 local nodes")
        assert {"compact_flat1", "hist8", "scan8"} <= chain, chain


def test_shard_status_words_do_not_alias_after_1024_calls(pkg, oracle):
    """A compaction tile accepts a predecessor's status word by its 10-bit epoch.  A large call, 1,023 one-tile calls, then a
    large call of the same size on other claims: the last call's epoch equals the first's modulo 1,024, and its tiles must
    not take the words the first call left as their own.  Without the clear at the epoch wrap this fails only when a tile
    reads a predecessor before that predecessor has published in the last call, which is likely with hundreds of tiles in
    flight but not certain; with it the test passes deterministically."""
    n = 200_000                                                         # 782 tiles of 256 claims
    x = pkg.synth.mixed(n, 400, 54, invalid=True)
    y = pkg.synth.mixed(n, 400, 55, invalid=True)
    y.claims["node"] = np.where(y.claims["node"] < 400, (y.claims["node"].astype(np.int64) ** 2) % 400, y.claims["node"]).astype(np.uint32)
    y.out_off, y.n_out = pkg.records.out_offsets(y.claims, y.n_node)
    y.gpus, y.node_off = x.gpus, x.node_off                            # same inventory, different per-tile counts
    small = pkg.synth.mixed(200, 400, 56, invalid=True)
    with pkg.api.Context(device=0) as c:
        c.set_table(x.table); c.set_inventory(x.gpus, x.node_off); c.set_shard(0, 200, take_stray=True)
        rx, rx_inv = oracle.allocate(x.gpus, x.node_off, x.table, x.claims, x.out_off, x.n_out, threads=8)
        dx, ox = S.dev(x.claims), S.dev(x.out_off)
        S.shard_call(pkg, c, x, dx, ox, 0, 200, True, rx, rx_inv, "first large call")
        ds, os_ = S.dev(small.claims), S.dev(small.out_off)
        for _ in range(1_023):
            c.allocate_global_device(ds.data_ptr(), small.n_claim, os_.data_ptr(), small.n_out, pkg.api.F_FRESH_INVENTORY)
        c.sync()
        ry, ry_inv = oracle.allocate(y.gpus, y.node_off, y.table, y.claims, y.out_off, y.n_out, threads=8)
        dy, oy = S.dev(y.claims), S.dev(y.out_off)
        _, _, chain = S.shard_call(pkg, c, y, dy, oy, 0, 200, True, ry, ry_inv, "large call 1,024 epochs later")
        assert "compact_flat1" in chain


# (A LARGE sharded batch across ranks — stand-alone gather after wave-sized hist tiles and the row-wise scan — is checked on
#  real ranks only: tests/multi_gpu_check.py, "1M claims x 10k nodes".  Two world contexts on ONE device cannot run it: a
#  rank's gather kernel holds every SM at the default shared-memory split while it waits for its peer, whose histogram CTAs
#  need the SMs re-split.  The compaction forms themselves are covered above on world-1 contexts, which have no gather.)
