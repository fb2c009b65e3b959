"""GPU suite: Deallocate on one inventory (dra_deallocate_batch, spec §9) at its edges.  Every call is compared byte for
byte with the CPU oracle, whose §9 is pinned to a plain restatement by tests/test_dealloc_oracle.py.  After each call the
pristine inventory must be as loaded: a DRA_F_FRESH_INVENTORY Allocate of one INVALID claim makes the live inventory the
pristine one, and get_inventory must then read the loaded bytes.  The records are arbitrary, not only ones Allocate
wrote: start and size up to 255, any status, GPU indices past the inventory, share counts and free memory that wrap."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import shard_world as S
from test_dealloc_oracle import BAD_RANGES, bad_range, releases

pytestmark = pytest.mark.gpu


def _ctx(pkg, gpus, node_off, flags=0):
    c = pkg.api.Context(device=0, flags=flags)
    c.set_table(pkg.records.default_table())
    c.set_inventory(gpus, node_off)
    return c


def _release(pkg, oracle, c, state, claims, out, out_off, n_node, what):
    """One dra_deallocate_batch on the live inventory `state`: one launch, and the oracle's inventory after it."""
    want = oracle.deallocate(state, claims, out, out_off, n_node=n_node)
    l0 = c.launch_count()
    c.deallocate(claims, out, out_off)
    assert c.launch_count() - l0 == (1 if len(claims) else 0), f"{what}: launches"
    got = c.get_inventory()
    if got.tobytes() != want.tobytes():
        bad = np.nonzero((got.view(np.uint8).reshape(-1, 16) != want.view(np.uint8).reshape(-1, 16)).any(1))[0]
        raise AssertionError(f"{what}: {len(bad)} GPUs differ from the oracle, first {bad[0]}: "
                             f"got {got[bad[0]]}, want {want[bad[0]]}")
    return want


def _pristine(pkg, c, loaded, what):
    """The pristine inventory is still the loaded one (this makes it the live one again)."""
    if len(loaded) == 0:
        return
    bad = np.zeros(1, dtype=pkg.records.CLAIM_DTYPE)
    bad["kind"] = 7                                              # INVALID: takes nothing
    c.allocate(bad, None, 1, pkg.api.F_FRESH_INVENTORY)
    assert c.get_inventory().tobytes() == loaded.tobytes(), f"{what}: the pristine inventory changed"


# ---- the CPU suite's problems on the device, on one inventory and sharded -------------------------------------------------
def test_hypothesis_problems_on_one_inventory_and_sharded(pkg, oracle):
    """releases() of the CPU suite: one reused context per call form.  The same garbage records go to the sharded call at
    worlds 1 to 4 (random bounds and stray rank), so both forms share §9's rule."""
    R = pkg.records
    big, big_off = R.make_inventory([9] * 4, mig=True)            # the generator's largest inventory: the sync's staging
    single = _ctx(pkg, big, big_off)
    worlds = {w: S.World(pkg, R.default_table(), big_off, big, w, S.bounds(4, w, "even")) for w in (1, 2, 3, 4)}
    try:
        @settings(max_examples=150, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True, database=None)
        @given(releases(), st.data())
        def run(prob, data):
            g, off, c, out, out_off = prob
            n_node = len(off) - 1
            single.set_inventory(g, off)
            _release(pkg, oracle, single, g, c, out, out_off, n_node, "one inventory")
            _pristine(pkg, single, g, "one inventory")
            if len(c) == 0:
                return
            want = oracle.deallocate(g, c, out, out_off, n_node=n_node)
            for w, W in worlds.items():
                cuts = sorted(data.draw(st.lists(st.integers(0, n_node), min_size=w - 1, max_size=w - 1)))
                bounds, stray = [0] + cuts + [n_node], data.draw(st.integers(0, w - 1))
                for x in W.ctxs:
                    x.set_inventory(g, off); x.set_shard_map(bounds, stray_rank=stray)
                W.node_off, W.n_node, W.bounds, W.loaded = off, n_node, bounds, [g] * w
                S.deallocate(W, c, out_off, len(out), want, f"world {w}, bounds {bounds}", out=out)
                W.assert_synced(want, f"world {w}, bounds {bounds}")
        run()
    finally:
        single.close()
        for W in worlds.values():
            W.close()


# ---- every (start, size) of a MIG record ----------------------------------------------------------------------------------
def test_every_start_and_size_in_one_call(pkg, oracle):
    """256 x 256 (start, size) pairs, one MIG GPU with every slice busy per pair, nodes of 32 GPUs, in one call.  The
    16-slice synthetic table's shapes (synth.homog(wide16=True)) free exactly their slices; a start of 16 or more frees
    none; a size of 16 or more frees everything from start up."""
    R = pkg.records
    n = 256 * 256
    gpus, node_off = R.make_inventory([32] * (n // 32), mig=True, busy=0xFFFF)
    claims = np.zeros(n, dtype=R.CLAIM_DTYPE)
    claims["kind"], claims["count"], claims["profile"] = R.KIND_MIG, 1, 1
    claims["node"] = np.arange(n) // 32
    out = np.zeros(n, dtype=R.OUT_DTYPE)
    out["gpu"] = np.arange(n)
    out["start"], out["size"] = np.arange(n) // 256, np.arange(n) % 256
    out["profile"], out["status"] = 1, R.ST_OK
    c = _ctx(pkg, gpus, node_off)
    try:
        want = _release(pkg, oracle, c, gpus, claims, out, None, len(node_off) - 1, "start/size grid")
        busy = want["busy"].reshape(256, 256).astype(np.int64)       # [start, size]
        shapes = [(1, s) for s in range(16)] + [(2, s) for s in range(0, 16, 2)] + [(5, s) for s in (0, 5, 10)] + \
                 [(8, 0), (8, 8), (16, 0)]
        for size, start in shapes:
            assert busy[start, size] == 0xFFFF & ~(((1 << size) - 1) << start), (start, size)
        assert (busy[16:, :] == 0xFFFF).all() and (busy[:, 0] == 0xFFFF).all()
        for start in range(16):
            assert (busy[start, 16:] == (1 << start) - 1).all(), start
        _pristine(pkg, c, gpus, "start/size grid")
    finally:
        c.close()


# ---- wrap and contention on one GPU word ----------------------------------------------------------------------------------
def test_wrap_and_contention_in_one_call(pkg, oracle):
    """One call, shuffled: 65,535 SHARED releases that take GPU 0's share_cnt from 0xFFFF to 0, 65,537 that wrap GPU 1's
    (3 to 2), 3 that take GPU 2's mem_free_mib past 2^32 and its share_cnt below 0, 16 one-slice releases of GPU 3, and
    a count-32 GPU claim over the 32 GPUs of node 1.  The rsvd words are non-zero, so a borrow out of share_cnt shows."""
    R = pkg.records
    rng = np.random.default_rng(7)
    gpus, node_off = R.make_inventory([4, 32], mig=False)
    gpus["share_cnt"][:3] = [0xFFFF, 3, 1]
    gpus["mem_free_mib"][:3] = [0, 0, 0xFFFFFF00]
    gpus["rsvd"] = 0x5A5A
    gpus["flags"][3], gpus["busy"][3] = R.GPU_MIG_ENABLED, 0xFFFF
    gpus["flags"][4:] = R.GPU_FULL_ALLOCATED
    kind = np.repeat(np.array([R.KIND_SHARED, R.KIND_SHARED, R.KIND_SHARED, R.KIND_MIG]), [65_535, 65_537, 3, 16])
    gpu = np.repeat(np.arange(4), [65_535, 65_537, 3, 16])
    mem = np.repeat(np.array([1, 2, 0x60000000, 0]), [65_535, 65_537, 3, 16])
    start = np.concatenate([np.zeros(65_535 + 65_537 + 3, dtype=np.int64), np.arange(16)])
    n = len(kind) + 1                                             # and claim n - 1: the count-32 GPU claim
    claims = np.zeros(n, dtype=R.CLAIM_DTYPE)
    claims["kind"][:-1], claims["count"][:-1], claims["mem_limit_mib"][:-1] = kind, 1, mem
    claims["profile"][:-1] = np.where(kind == R.KIND_MIG, 1, 0)
    claims[-1] = (R.KIND_GPU, 0, 32, 1, 0, 0)
    perm = rng.permutation(n)                                     # the order the claims take their slots in
    sl = np.where(np.arange(n) == n - 1, 32, 1)[perm]
    out_off = np.zeros(n, dtype=np.uint32)
    out_off[perm] = np.cumsum(sl) - sl
    out = np.zeros(n + 31, dtype=R.OUT_DTYPE)
    o = out_off[:-1].astype(np.int64)
    out["gpu"][o], out["start"][o] = gpu, start
    out["size"][o] = np.where(kind == R.KIND_MIG, 1, 0)
    out["profile"][o] = np.where(kind == R.KIND_MIG, 1, R.PROFILE_SHARED)
    g0 = int(out_off[-1])
    out["gpu"][g0: g0 + 32], out["profile"][g0: g0 + 32] = np.arange(4, 36), R.PROFILE_GPU
    out["status"] = R.ST_OK
    c = _ctx(pkg, gpus, node_off)
    try:
        want = _release(pkg, oracle, c, gpus, claims, out, out_off, 2, "wrap and contention")
        assert list(want["share_cnt"][:3]) == [0, 2, 0xFFFE]
        assert list(want["mem_free_mib"][:3]) == [65_535, 2 * 65_537, (0xFFFFFF00 + 3 * 0x60000000) % (1 << 32)]
        assert want["busy"][3] == 0 and not (want["flags"][4:] & R.GPU_FULL_ALLOCATED).any()
        assert (want["rsvd"] == 0x5A5A).all()
        _pristine(pkg, c, gpus, "wrap and contention")
    finally:
        c.close()


# ---- the one-thread-per-claim grid at its edges ---------------------------------------------------------------------------
def _host_free():
    try:
        with open("/proc/meminfo") as f:
            return next(int(x.split()[1]) * 1024 for x in f if x.startswith("MemAvailable"))
    except (OSError, StopIteration):
        return 0


def _need(dev_bytes, host_bytes):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < dev_bytes:
        pytest.skip(f"needs {dev_bytes / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free")
    if _host_free() < host_bytes:
        pytest.skip(f"needs {host_bytes / 2**30:.1f} GiB of host memory, {_host_free() / 2**30:.1f} GiB available")


def _mixed_records(R, rng, n_claim, n_node, per_node):
    """n_claim claims of every kind over a taken inventory, with out_off; records of any status, GPU indices up to 8 past
    the inventory.  The SHARED releases spread over every GPU, so no word takes more than a few hundred atomics."""
    gpus, node_off = R.make_inventory([per_node] * n_node, mig=True, busy=0xFFFF)
    n_gpu = len(gpus)
    gpus["flags"][::2] = R.GPU_FULL_ALLOCATED
    gpus["share_cnt"], gpus["mem_free_mib"] = 0x4000, 0xFFFF0000
    c = np.zeros(n_claim, dtype=R.CLAIM_DTYPE)
    c["kind"] = rng.integers(0, 5, n_claim)
    c["node"] = np.where(rng.random(n_claim) < 0.05, n_node, rng.integers(0, n_node, n_claim))
    c["count"] = np.where(c["kind"] == R.KIND_GPU, rng.choice(np.array([0, 1, 2, 32, 33]), n_claim), 1)
    c["mem_limit_mib"] = rng.integers(0, 1 << 20, n_claim)
    out_off, n_out = R.out_offsets(c, n_node)
    out = np.zeros(int(n_out), dtype=R.OUT_DTYPE)
    out["gpu"] = rng.integers(0, n_gpu + 8, int(n_out))
    out["start"], out["size"] = rng.integers(0, 20, int(n_out)), rng.choice(np.array([1, 2, 4, 8, 16, 32, 255]), int(n_out))
    out["status"] = np.where(rng.random(int(n_out)) < 0.85, R.ST_OK, rng.integers(1, 256, int(n_out)))
    return gpus, node_off, c, out_off, out


@pytest.mark.parametrize("n_claim", [1, 255, 256, 257, (1 << 22) + 1])
def test_grid_edges(pkg, oracle, n_claim):
    """n_claim at one CTA's edges and at about 4M claims (16,385 CTAs, 64 MB of claims)."""
    R = pkg.records
    if n_claim > 1 << 20:
        _need(1 << 30, 4 << 30)
    rng = np.random.default_rng(n_claim)
    gpus, node_off, claims, out_off, out = _mixed_records(R, rng, n_claim, 128, 32)
    c = _ctx(pkg, gpus, node_off)
    try:
        _release(pkg, oracle, c, gpus, claims, out, out_off, 128, f"{n_claim} claims")
        _pristine(pkg, c, gpus, f"{n_claim} claims")
    finally:
        c.close()


# ---- a bad slot range changes nothing ---------------------------------------------------------------------------------
@pytest.mark.parametrize("where", BAD_RANGES)
def test_bad_slot_range_changes_nothing(pkg, oracle, where):
    """A slot range past n_out (first, middle or last claim with out_off, one at 0xFFFFFFFF, or n_out < n_claim without
    out_off): DRA_E_INVAL, no launch, the live and pristine inventories unchanged.  The next call on the context works."""
    api = pkg.api
    g, claims, out, out_off, keep = bad_range(where)
    node_off = np.array([0, len(g)], dtype=np.uint32)
    c = _ctx(pkg, g, node_off)
    try:
        state = _release(pkg, oracle, c, g, claims[:1], out, None, 1, "a first release")   # live differs from pristine
        l0 = c.launch_count()
        with pytest.raises(api.DraError) as e:
            c.deallocate(claims, out, out_off)
        assert e.value.code == api.E_INVAL
        assert c.launch_count() == l0, "a refused Deallocate launched a kernel"
        assert c.get_inventory().tobytes() == state.tobytes(), "a refused Deallocate changed the live inventory"
        _release(pkg, oracle, c, state, claims[keep], out, None if out_off is None else out_off[keep], 1, "the next call")
        _pristine(pkg, c, g, where)
    finally:
        c.close()


# ---- release part of an Allocate, then Allocate again, on every chain -------------------------------------------------
# the context's flags, and what the chain of kernels an Allocate took must satisfy
FUSED = {"fused_direct", "fused_staged", "fused_stream"}
CHAINS = {"direct": ((), lambda ch: "fused_direct" in ch),
          "nodirect": (("CFG_NO_DIRECT",), lambda ch: "fused_staged" in ch),
          "nofused": (("CFG_NO_FUSED",), lambda ch: ch and not ch & (FUSED | {"serve"})),
          "graph": (("CFG_USE_GRAPH", "CFG_NO_DIRECT"), lambda ch: ch and not ch & {"fused_direct", "serve"}),
          "resident": (("CFG_RESIDENT",), lambda ch: ch == {"serve"})}


@pytest.mark.parametrize("chain", list(CHAINS))
def test_release_a_subset_then_allocate(pkg, oracle, chain, request):
    """An Allocate, then a third of its claims released in reverse order and another third shuffled, each call checked;
    then two more Allocates, whose OutRecs must be the oracle's on the released state, and which take GPUs the releases
    freed."""
    R, api = pkg.records, pkg.api
    flags, want_chain = CHAINS[chain]
    rng = np.random.default_rng(len(chain))
    w = pkg.synth.mixed(1500, 17, 40 + len(chain), invalid=True)
    batches = [w.claims] + [pkg.synth.mixed(1500, 17, 50 + k + len(chain), invalid=True).claims for k in range(2)]
    c = pkg.api.Context(device=0, flags=sum(getattr(api, f) for f in flags))
    pins = None
    if chain == "resident":
        n_o = max(int(R.out_offsets(b, w.n_node)[1]) for b in batches)
        pins = [api.PinnedBuffer(1500, R.CLAIM_DTYPE), api.PinnedBuffer(1500, np.uint32), api.PinnedBuffer(n_o, R.OUT_DTYPE)]
        for b in pins:
            request.addfinalizer(b.free)
    try:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        state = w.gpus

        def alloc(claims, what):
            nonlocal state
            oo, n_out = R.out_offsets(claims, w.n_node)
            ref, state = oracle.allocate(state, w.node_off, w.table, claims, oo, n_out)
            if pins:
                n = len(claims)
                pins[0].array[:n], pins[1].array[:n] = claims, oo
                got = c.allocate(pins[0].array[:n], pins[1].array[:n], n_out, out=pins[2].array[:n_out]).copy()
            else:
                got = c.allocate(claims, oo, n_out)
            assert got.tobytes() == ref.tobytes(), f"{chain} {what}: OutRecs differ from the oracle"
            assert c.get_inventory().tobytes() == state.tobytes(), f"{chain} {what}: inventory differs from the oracle"
            assert want_chain(c.last_chain()), f"{chain} {what}: took {sorted(c.last_chain())}"
            return ref, oo

        ref, oo = alloc(batches[0], "first Allocate")
        sel = rng.permutation(len(batches[0]))
        sl = R.claim_slots(batches[0], w.n_node)
        freed = set()
        for part, what in ((np.sort(sel[:500])[::-1], "reverse"), (sel[500:1000], "shuffled")):
            before = state
            state = _release(pkg, oracle, c, state, batches[0][part], ref, oo[part], w.n_node, f"{chain} {what} release")
            assert state.tobytes() != before.tobytes(), f"{chain} {what} release: nothing was released"
            freed |= {int(ref["gpu"][int(oo[i]) + k]) for i in part for k in range(int(sl[i]))
                      if ref["status"][int(oo[i]) + k] == R.ST_OK}
        taken = set()
        for k in (1, 2):
            got = alloc(batches[k], f"Allocate {k} after the releases")[0]
            taken |= set(got["gpu"][got["status"] == R.ST_OK].tolist())
        assert freed & taken, f"{chain}: no GPU the releases freed was taken again"
        _pristine(pkg, c, w.gpus, chain)
    finally:
        c.close()
