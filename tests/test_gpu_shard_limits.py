"""GPU suite: the sharded Allocate (dra_allocate_batch_global_device) at the record limits, with selectors, on every chain a
shard can take, byte for byte against the oracle on the whole batch.  The problems are tests/shard_limit_problems.py's
(test_gpu_limits.py's seeds and fixtures, synth.mixed with selectors, one-node packet fixtures):
  form a   worlds of 1-4 contexts on one device, both ownership forms (dra_set_shard_map: every rank counts every rank's
           slots; bare dra_set_shard: the counts travel in a header) and both slot forms (out_off; none, n_out = n_claim).
           Every rank's gathered table is the oracle's, every rank's own GPU range the oracle's inventory, the chain is the
           compaction plus the single-launch kernel with its gather tail.  A second call without F_FRESH_INVENTORY answers
           as the oracle does on the first call's state; the sharded Deallocate of both gathered tables, in reverse order,
           gives every rank's own range back pristine, and after the inventory sync every rank holds the pristine inventory.
  form b   world-1 sub-range shards between an empty node 0 and a node outside the shard, padded with dropped claims past
           each compaction and chain limit; the kept slots and the shard's inventory are the oracle's, no other GPU changes.
(Worlds above 1 run only problems the default plan sends through the single-launch kernel with its gather tail: the end
of test_gpu_shard.py says why two world contexts on one device cannot run the stand-alone gather after a large kernel.)"""
import numpy as np
import pytest

import shard_limit_problems as SP
from test_gpu_limits import ONE_WAVE_FUSED_MAX, _sms
from test_gpu_paths import SORT8, STAGED_CAP, assert_same
import shard_world as S

pytestmark = pytest.mark.gpu

R = SP.R
N_OUT_MAX = 1 << 16                      # the exported table: far above every n_out here (the padding check needs 64)
TAIL = {"compact_flat1", "fused_staged"}


class ShardWorld(S.World):
    """A world exported once for an inventory of 256 GPUs; load() puts any smaller problem on it."""

    def __init__(self, pkg, world):
        g, off = R.make_inventory([32] * 8, mig=True)
        super().__init__(pkg, R.default_table(), off, g, world, [8 * r // world for r in range(world)] + [8],
                         n_out_max=N_OUT_MAX)

    def load(self, w, bounds, stray_rank, mapped):
        self.node_off, self.n_node, self.loaded, self.bounds = w.node_off, len(w.node_off) - 1, [w.gpus] * self.world, list(bounds)
        attrs = getattr(w, "attrs", None)
        for r, c in enumerate(self.ctxs):
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
            c.set_gpu_attrs(attrs); c.set_selectors(None if attrs is None else w.sels.reshape(-1, R.SEL_MAX_INS))
            if mapped:
                c.set_shard_map(bounds, stray_rank=stray_rank)
            else:
                c.set_shard(bounds[r], bounds[r + 1], take_stray=r == stray_rank)

    def sharded(self, d_claims, d_off, n_claim, n_out, flags, ref, state, what):
        """One call on every rank: every rank's table and own range against the oracle, nothing written outside the range,
        the compaction and the single-launch kernel (with its gather tail: two launches) taken."""
        import torch
        torch.cuda.synchronize()
        before, l0 = self.inventories(), [c.launch_count() for c in self.ctxs]
        for c in self.ctxs:
            c.allocate_global_device(d_claims.data_ptr(), n_claim, None if d_off is None else d_off.data_ptr(), n_out, flags)
        for c in self.ctxs:
            c.sync()
        tables = []
        for r, (c, b) in enumerate(zip(self.ctxs, before)):
            got = c.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE))
            inv = c.get_inventory()
            g0, g1 = self.gpu_range(r)
            assert_same(got, inv[g0:g1], ref, state[g0:g1], f"{what}: rank {r}")
            assert inv[:g0].tobytes() == b[:g0].tobytes() and inv[g1:].tobytes() == b[g1:].tobytes(), \
                f"{what}: rank {r} wrote GPUs outside its range"
            assert c.last_chain() == TAIL and c.launch_count() - l0[r] == 2, \
                f"{what}: rank {r} took {sorted(c.last_chain())} in {c.launch_count() - l0[r]} launches"
            tables.append(got)
        return tables


@pytest.fixture(scope="module")
def worlds(pkg):
    ws = {k: ShardWorld(pkg, k) for k in (1, 2, 3, 4)}
    yield ws
    for W in ws.values():
        W.close()


def run_form_a(pkg, oracle, W, w, bounds, stray, mapped, slot, what):
    """Form a on world W: a fresh call, a call on its state, both released in reverse order, then the sync."""
    out_off, n_out = SP.slot_form(w, slot)
    world = len(W.ctxs)
    W.load(w, bounds, stray, mapped)
    d_c, d_o = S.dev(w.claims), None if out_off is None else S.dev(out_off)
    ref1, s1 = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, out_off, n_out)
    t1 = W.sharded(d_c, d_o, w.n_claim, n_out, pkg.api.F_FRESH_INVENTORY, ref1, s1, what)
    # the first call's gathered tables, kept for the release (world 1 has one table, which the next call overwrites)
    keep = [S.dev(t) for t in t1] if world == 1 else None
    p1 = [k.data_ptr() for k in keep] if world == 1 else [S.table_ptr(c) for c in W.ctxs]
    ref2, s2 = oracle.allocate(s1, w.node_off, w.table, w.claims, out_off, n_out)
    W.sharded(d_c, d_o, w.n_claim, n_out, 0, ref2, s2, f"{what}, second call")
    p2 = [S.table_ptr(c) for c in W.ctxs]
    assert world == 1 or not set(p1) & set(p2), "the two calls' tables share a buffer"
    st = oracle.deallocate(s2, w.claims, ref2, out_off, n_node=w.n_node)
    S.deallocate(W, w.claims, out_off, n_out, st, f"{what}: release of the second call", ptrs=p2)
    st = oracle.deallocate(st, w.claims, ref1, out_off, n_node=w.n_node)
    assert st.tobytes() == w.gpus.tobytes(), f"{what}: the oracle does not release to pristine"
    S.deallocate(W, w.claims, out_off, n_out, st, f"{what}: release of the first call", ptrs=p1)
    del keep
    if world > 1:
        if not mapped:
            W.remap(bounds, stray)                        # the sync needs every rank's range
        W.assert_synced(w.gpus, f"{what}: after the sync")
    return ref1


FORMS_A = [(world, mapped) for world in (1, 2, 3, 4) for mapped in (True, False)]


@pytest.mark.parametrize("world,mapped", FORMS_A, ids=[f"world{k}-{'map' if m else 'bare'}" for k, m in FORMS_A])
def test_limit_problems_on_worlds(pkg, oracle, worlds, world, mapped):
    W = worlds[world]
    n = 0
    for w in SP.problems():
        for k, bounds, stray in SP.splits(w):
            if k != world:
                continue
            for slot in ("off", "nooff"):
                run_form_a(pkg, oracle, W, w, bounds, stray, mapped, slot, f"{w.name}, bounds {bounds}, strays on {stray}, {slot}")
                n += 1
    assert n


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_selectors_on_worlds(pkg, oracle, worlds, world):
    """synth.with_selectors' table and seeded random programs; the GPU claim of count 3 naming the id beyond the table keeps
    its three slots, all INVALID, in every rank's table."""
    W = worlds[world]
    beyond_elsewhere = 0
    for seed in SP.SEL_SEEDS:
        w = SP.selector_problem(seed)
        oracle.set_selectors(w.attrs, w.sels)
        try:
            for k, bounds, stray in SP.selector_splits(w):
                if k != world:
                    continue
                for mapped in (True, False):
                    ref = run_form_a(pkg, oracle, W, w, bounds, stray, mapped, "off",
                                     f"{w.name}, bounds {bounds}, strays on {stray}, {'map' if mapped else 'bare'}")
                    o = int(w.out_off[w.beyond])
                    assert (ref["status"][o: o + 3] == R.ST_INVALID).all() and int(w.out_off[w.beyond + 1]) == o + 3
                    beyond_elsewhere += int(SP.owner(w.claims[w.beyond: w.beyond + 1], w.n_node, bounds, stray)[0] != stray)
        finally:
            oracle.set_selectors()
    assert world == 1 or beyond_elsewhere, "the claim beyond the table never sat on a non-stray rank"


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("name", SP.PACKET_FIXTURES)
def test_packet_fixtures(pkg, oracle, worlds, world, name):
    """The only node on the last rank, the strays on rank 0: records at the top of every packet field cross to every rank."""
    w = SP.packet_fixture(name)
    ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    assert SP.PACKET_EXPECT[name](ref), ref
    bounds = [0] * world + [1]
    for mapped in (True, False):
        for slot in ("off", "nooff"):
            run_form_a(pkg, oracle, worlds[world], w, bounds, 0, mapped, slot, f"{name}, world {world}, {slot}")


class _Raw:
    """A device range as a torch tensor (__cuda_array_interface__), to write and read a gathered table's padding."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


@pytest.mark.parametrize("world", [2, 4])
def test_gathered_table_padding_is_left_alone(pkg, oracle, worlds, world):
    """Both parity tables carry a sentinel in [n_out, n_out_max); two further calls write only [0, n_out) of them."""
    import torch
    W = worlds[world]
    w = SP.packet_fixture("statuses")
    assert N_OUT_MAX >= w.n_out + 64
    W.load(w, [0] * world + [1], 0, True)
    d_c, d_o = S.dev(w.claims), S.dev(w.out_off)
    ref, st = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    ptrs = []
    for k in range(2):
        W.sharded(d_c, d_o, w.n_claim, w.n_out, pkg.api.F_FRESH_INVENTORY, ref, st, f"call {k}")
        ptrs.append([S.table_ptr(c) for c in W.ctxs])
    pads = [torch.as_tensor(_Raw(p + 8 * w.n_out, 8 * (N_OUT_MAX - w.n_out)), device="cuda:0") for ps in ptrs for p in ps]
    assert len({p for ps in ptrs for p in ps}) == 2 * world
    for t in pads:
        t.fill_(0xA5)
    torch.cuda.synchronize()
    for k in range(2):
        W.sharded(d_c, d_o, w.n_claim, w.n_out, pkg.api.F_FRESH_INVENTORY, ref, st, f"call {k + 2}")
    torch.cuda.synchronize()
    for i, t in enumerate(pads):
        assert bool((t == 0xA5).all()), f"table {i}: the padding past n_out was written"


# ---- form b: world-1 sub-range shards -----------------------------------------------------------------------------------
def _form_b(pkg, oracle, v, first, hinted, what, flags=0):
    """Two calls of v on a world-1 shard [v.lo, v.hi) with strays: the first call's chain passes `first`, the second (the
    plan from the first call's count) `hinted`; kept slots and the shard's GPUs against the oracle, no other GPU changed."""
    ref, ref_inv = oracle.allocate(v.gpus, v.node_off, v.table, v.claims, v.out_off, v.n_out, threads=8)
    with pkg.api.Context(device=0, flags=flags) as c:
        c.set_table(v.table); c.set_inventory(v.gpus, v.node_off)
        attrs = getattr(v, "attrs", None)
        if attrs is not None:
            c.set_gpu_attrs(attrs); c.set_selectors(v.sels.reshape(-1, R.SEL_MAX_INS))
        c.set_shard(v.lo, v.hi, take_stray=True)
        d, o = S.dev(v.claims), S.dev(v.out_off)
        for k, want in enumerate((first, hinted)):
            if want is None:
                continue
            _, _, chain = S.shard_call(pkg, c, v, d, o, v.lo, v.hi, True, ref, ref_inv, f"{what}, call {k}")
            assert want(chain) if callable(want) else chain == want, f"{what}, call {k}: took {sorted(chain)}"
            g0, g1 = int(v.node_off[v.lo]), int(v.node_off[v.hi])
            inv = c.get_inventory()
            assert inv[:g0].tobytes() == v.gpus[:g0].tobytes() and inv[g1:].tobytes() == v.gpus[g1:].tobytes(), \
                f"{what}: a GPU outside the shard changed"


PADDED = {   # padded to, chain of the first call, chain of the call planned from its count
    "stream": (STAGED_CAP + 1, {"compact_flat1", "fused_stream"}, {"compact_flat1", "fused_staged"}),
    "sort": (ONE_WAVE_FUSED_MAX + 1, {"compact_flat1", "pack1"} | SORT8, {"compact_flat1", "fused_staged"}),
    "flat8": (262_145, lambda ch: "compact_flat8" in ch, {"compact_flat8", "fused_staged"}),
    "lookback": (2_097_153, lambda ch: "compact_lookback" in ch, {"compact_lookback", "fused_staged"}),
}


@pytest.mark.parametrize("form", list(PADDED))
def test_limit_problems_padded_on_a_shard(pkg, oracle, form):
    n_total, first, hinted = PADDED[form]
    probs = SP.problems()
    for w in probs[:6] if form == "lookback" else probs:
        _form_b(pkg, oracle, SP.padded(w, n_total), first, hinted, f"{w.name} padded to {n_total}")


def test_limit_problems_on_a_shard_sort_chain(pkg, oracle):
    """CFG_NO_FUSED: the one-CTA counting sort and a warp per node under the shard's view."""
    for w in SP.problems():
        v = SP.padded(w, SP.SORT_CHAIN_PAD(w))
        _form_b(pkg, oracle, v, {"compact_flat1", "bucket_small", "pack1"}, None, f"{w.name}, no fused kernel",
                flags=pkg.api.CFG_NO_FUSED)


def test_limit_problems_tiled_on_a_shard_pack4(pkg, oracle):
    """More local nodes than k_pack<1> serves (16 per SM), fewer than the sharded call's 12,798: warps of k_pack<4>."""
    S = _sms()
    for w in SP.problems()[:6]:
        v = SP.tiled(w, 16 * S + 1)
        assert 16 * S < v.hi - v.lo <= 12_798
        _form_b(pkg, oracle, v, lambda ch: "pack4" in ch and not ch & {"fused_staged", "fused_stream"}, None,
                f"{w.name} over {v.hi - v.lo} nodes")


@pytest.mark.parametrize("form", ["stream", "flat8", "lookback"])
def test_selectors_padded_on_a_shard(pkg, oracle, form):
    n_total, first, hinted = PADDED[form]
    seeds = SP.SEL_SEEDS[:2] if form == "lookback" else SP.SEL_SEEDS
    for seed in seeds:
        w = SP.selector_problem(seed)
        v = SP.padded(w, n_total)
        oracle.set_selectors(v.attrs, v.sels)
        try:
            _form_b(pkg, oracle, v, first, hinted, f"{w.name} padded to {n_total}")
        finally:
            oracle.set_selectors()
