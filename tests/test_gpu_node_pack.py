"""GPU suite: the single-launch Allocate kernel's node-wide pack, on both sides of its selection, bit-exact with the oracle.

A node's claims take the node-wide pack (every thread prepares one record, warp 0 runs one loop over all of them, every
thread stores one OutRec) when the node is homogeneous, every claim of it is a plain MIG claim (valid profile, no selector,
no co-location group, its slot in range) and the node has at most as many claims as the prepared-record area holds:
min(256, index-list bytes / 36).  Every other node keeps the per-segment pack.  Each batch below mixes nodes of both kinds,
and every case runs on the staged and streamed layouts, with and without out_off, through the launched kernel, direct
host I/O and the resident kernel.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NW, PIECE = 8, 256                                  # warps per CTA; claims per staged piece
STAGED_CAP = 11_117


def area_limit(n_claim):
    """Most claims of one node the node-wide pack takes in a batch of n_claim claims (staged layout)."""
    chunk = -(-n_claim // (NW * PIECE)) * PIECE
    return min(NW * 32, chunk * NW * 4 // 36)


def _inventory(R, n_node, rng, hetero=(), rough=False):
    g, off = R.make_inventory([8] * n_node, mig=True)
    if rough:                                       # occupied slices, unavailable and MIG-disabled GPUs
        g["busy"] = np.where(rng.integers(0, 3, len(g)) == 0, rng.integers(0, 256, len(g)), 0).astype(np.uint16)
        g["flags"] |= np.where(rng.integers(0, 13, len(g)) == 0, R.GPU_UNAVAILABLE, 0).astype(np.uint8)
        g["flags"] &= np.where(rng.integers(0, 11, len(g)) == 0, ~np.uint8(R.GPU_MIG_ENABLED), 0xFF).astype(np.uint8)
    for n in hetero:                                # a node with a GPU of the 4-slice model
        g["model"][off[n] + 3] = 1
    return g, off


def _claims(R, counts, rng, profs=(0, 0, 0, 0, 1, 1, 1, 2, 2, 4)):
    """counts[n] plain MIG claims on node n, 1g/2g/3g/7g 40/30/20/10 %, interleaved at random over the batch."""
    node = np.repeat(np.arange(len(counts), dtype=np.uint32), counts)
    rng.shuffle(node)
    c = np.zeros(len(node), dtype=R.CLAIM_DTYPE)
    c["kind"] = R.KIND_MIG
    c["count"] = 1
    c["node"] = node
    c["profile"] = np.array(profs, dtype=np.uint8)[rng.integers(0, len(profs), len(node))]
    return c


def _claims_of(c, n):
    return np.nonzero(c["node"] == n)[0]


def batch(pkg, kind, seed):
    """(gpus, node_off, table, claims, n_node): the nodes of one case."""
    R = pkg.records
    rng = np.random.default_rng(seed)
    t = R.default_table()
    if kind == "limits_small":                      # <= 2048 claims: the area holds 227 records
        lim = area_limit(2048)
        assert lim == 227
        counts = [1, 2, 31, 32, 33, 64, 65, lim - 1, lim, lim + 1]
        g, off = _inventory(R, len(counts), rng)
        c = _claims(R, counts, rng)
    elif kind == "limits_large":                    # > 2048 claims: 256 records, one per thread
        counts = [255, 256, 257] + [80] * 17
        assert area_limit(sum(counts)) == 256
        g, off = _inventory(R, len(counts), rng, rough=True)
        c = _claims(R, counts, rng)
    elif kind == "one_other":                       # one claim of the node is not a plain MIG claim
        counts = [80] * 12
        g, off = _inventory(R, len(counts), rng)
        c = _claims(R, counts, rng)
        for n, (field, val), at in [(1, ("kind", R.KIND_GPU), 0), (2, ("kind", R.KIND_SHARED), 40),
                                    (3, ("group", 1), 79), (4, ("profile", 16), 10), (5, ("profile", 0xFE), 79)]:
            i = _claims_of(c, n)[at]
            c[field][i] = val
            if field == "kind" and val == R.KIND_SHARED:
                c["mem_limit_mib"][i] = 1024
    elif kind == "hetero":                          # one GPU of another model: per-GPU table rows
        counts = [80, 80, 80, 80]
        g, off = _inventory(R, len(counts), rng, hetero=(1, 3))
        c = _claims(R, counts, rng)
    elif kind == "all_die":                         # every shape dies well before the end of the node's list
        counts = [120, 200, 90, 150]
        g, off = _inventory(R, len(counts), rng)
        c = _claims(R, counts, rng)
        for n in range(len(counts)):                # the node fills up with 1g first, then every shape fails
            i = _claims_of(c, n)
            c["profile"][i[:60]] = R.GI_1_SLICE
            c["profile"][i[60:]] = np.array([R.GI_1_SLICE, R.GI_2_SLICE, R.GI_3_SLICE, R.GI_7_SLICE],
                                            dtype=np.uint8)[np.arange(len(i) - 60) % 4]
        c["profile"][_claims_of(c, 2)[:3]] = R.GI_7_SLICE     # 7g dies inside the first record pair on node 2
    elif kind == "dead_early":                      # shapes die one by one while others still fit
        counts = [100, 100, 100]
        g, off = _inventory(R, len(counts), rng, rough=True)
        c = _claims(R, counts, rng, profs=(4, 4, 2, 1, 0))
    else:
        raise AssertionError(kind)
    return g, off, t, c, len(counts)


def streamed(pkg, w):
    """The same nodes in a batch too large to stage: filler claims naming no node pad it past the staged capacity."""
    R = pkg.records
    g, off, t, c, n_node = w
    pad = np.zeros(STAGED_CAP + 1 - len(c), dtype=R.CLAIM_DTYPE)
    pad["kind"] = R.KIND_MIG
    pad["count"] = 1
    pad["node"] = n_node + 7
    allc = np.concatenate([c, pad])
    np.random.default_rng(5).shuffle(allc)
    return g, off, t, allc, n_node


CASES = ["limits_small", "limits_large", "one_other", "hetero", "all_die", "dead_early"]
CTX = {"launch": "nodirect", "direct": 0, "resident": "resident"}


def _flags(pkg, name):
    return {0: 0, "nodirect": pkg.api.CFG_NO_DIRECT, "resident": pkg.api.CFG_RESIDENT}[name]


@pytest.mark.parametrize("layout", ["staged", "streamed"])
@pytest.mark.parametrize("with_off", [False, True])
@pytest.mark.parametrize("path", list(CTX))
@pytest.mark.parametrize("kind", CASES)
def test_node_pack_matches_oracle(pkg, oracle, kind, path, with_off, layout):
    if layout == "streamed" and path != "launch":
        pytest.skip("batches past the staged capacity take the launched kernel only")
    R = pkg.records
    w = batch(pkg, kind, seed=CASES.index(kind) + 31)
    if layout == "streamed":
        w = streamed(pkg, w)
    g, off, t, c, n_node = w
    if with_off:
        out_off, n_out = R.out_offsets(c, n_node)
    else:
        out_off, n_out = None, len(c)
    ref_out, ref_inv = oracle.allocate(g, off, t, c, out_off, n_out, threads=8)
    with pkg.api.Context(device=0, flags=_flags(pkg, CTX[path])) as ctx:
        ctx.set_table(t)
        ctx.set_inventory(g, off)
        out = ctx.allocate(c, out_off, n_out)
        inv = ctx.get_inventory()
        chain = ctx.last_chain()
    want = {"staged": {"launch": {"fused_staged"}, "direct": {"fused_direct"}, "resident": {"serve"}},
            "streamed": {"launch": {"fused_stream"}}}[layout][path]
    assert chain == want, f"{kind}: took {sorted(chain)}"
    if out.tobytes() != ref_out.tobytes():
        bad = np.nonzero(out.view(np.uint64) != ref_out.view(np.uint64))[0]
        raise AssertionError(f"{kind}: {len(bad)} OutRecs differ, first at {bad[0]}: cuda={out[bad[0]]} oracle={ref_out[bad[0]]}")
    assert inv.tobytes() == ref_inv.tobytes(), f"{kind}: inventory differs from the oracle"


def test_cases_reach_the_area_limit(pkg):
    """The limit cases put nodes just under, at and just over the prepared-record area."""
    g, off, t, c, n_node = batch(pkg, "limits_small", 1)
    per_node = np.bincount(c["node"], minlength=n_node)
    assert per_node.max() == area_limit(len(c)) + 1 and (per_node == area_limit(len(c))).any()
    g, off, t, c, n_node = batch(pkg, "limits_large", 1)
    assert sorted(np.bincount(c["node"]))[-3:] == [255, 256, 257] and area_limit(len(c)) == 256


def test_node_pack_is_taken_where_selected(pkg, oracle, monkeypatch):
    """The node-wide pack runs on exactly the nodes its selection admits (read from the DRA_TIMELINE stamps: on that
    path the fetch and part-a fields of word 7 stay 0, and the count field is the node's claim count)."""
    monkeypatch.setenv("DRA_TIMELINE", "1")
    for kind, per_segment in [("limits_small", {9}), ("one_other", {1, 2, 3, 4, 5}), ("hetero", {1, 3})]:
        g, off, t, c, n_node = batch(pkg, kind, seed=CASES.index(kind) + 31)
        out_off, n_out = pkg.records.out_offsets(c, n_node)
        with pkg.api.Context(device=0, flags=pkg.api.CFG_NO_DIRECT) as ctx:
            ctx.set_table(t)
            ctx.set_inventory(g, off)
            out = ctx.allocate(c, out_off, n_out)
            tl = ctx.debug_timeline(n_node + 1)
        ref_out, _ = oracle.allocate(g, off, t, c, out_off, n_out, threads=8)
        assert out.tobytes() == ref_out.tobytes(), kind
        w7 = tl[:n_node, 7].astype(np.uint64)
        counts = np.bincount(c["node"], minlength=n_node)
        assert ((w7 & np.uint64(0xFFFF)) == counts).all(), kind
        node_wide = {n for n in range(n_node) if int(w7[n]) >> 32 == 0}
        assert node_wide == set(range(n_node)) - per_segment, f"{kind}: node-wide pack on {sorted(node_wide)}"


@pytest.mark.parametrize("path", ["launch", "direct"])
def test_out_of_range_slot_on_a_node_wide_node(pkg, path):
    """A claim whose out slot is past n_out, on a node that takes the node-wide pack: the call fails with the range error,
    and the claim takes no capacity — the inventory ends as the sort path (per-segment pack) leaves it."""
    R = pkg.records
    g, off, t, c, n_node = batch(pkg, "dead_early", seed=40)
    out_off, n_out = R.out_offsets(c, n_node)
    i = _claims_of(c, 1)[3]
    c["profile"][i] = R.GI_7_SLICE
    out_off = out_off.copy()
    out_off[i] = n_out
    invs = []
    for flags in (_flags(pkg, CTX[path]), pkg.api.CFG_NO_FUSED):
        with pkg.api.Context(device=0, flags=flags) as ctx:
            ctx.set_table(t)
            ctx.set_inventory(g, off)
            with pytest.raises(pkg.api.DraError):
                ctx.allocate(c, out_off, n_out)
            invs.append(ctx.get_inventory())
    assert invs[0].tobytes() == invs[1].tobytes()


def test_sharded_tail_on_per_segment_nodes(pkg, oracle):
    """A world of 2 whose fused calls end in the multi-GPU tail with its send queue: MIG-off nodes with 40 SHARED claims
    and heterogeneous nodes with 40 MIG claims (per-segment pack, a full first segment) beside node-wide nodes."""
    import shard_world as S
    R = pkg.records
    rng = np.random.default_rng(77)
    counts = [40, 40, 40, 40, 40, 40, 80, 80, 80, 80, 80, 40]
    g, off = _inventory(R, len(counts), rng, hetero=(4, 5))
    for n in range(4):                                  # MIG off
        g["flags"][off[n]:off[n + 1]] = 0
    c = _claims(R, counts, rng)
    sh = np.isin(c["node"], [0, 1, 2, 3])
    c["kind"][sh] = R.KIND_SHARED
    c["profile"][sh] = 0
    c["mem_limit_mib"][sh] = np.array([1024, 4096, 10240], dtype=np.uint32)[rng.integers(0, 3, int(sh.sum()))]
    n_node = len(counts)
    t = R.default_table()
    out_off, n_out = R.out_offsets(c, n_node)
    ref, ref_inv = oracle.allocate(g, off, t, c, out_off, n_out, threads=8)
    bounds = [0, n_node // 2, n_node]
    with S.World(pkg, t, off, g, 2, bounds, n_out_max=n_out) as W:
        for rep in range(3):
            tables = S.allocate(W, c, out_off, n_out, pkg.api.F_FRESH_INVENTORY)
            for r, got in enumerate(tables):
                assert got.tobytes() == ref.tobytes(), f"rank {r} call {rep}: table differs from the oracle"
            assert W.state().tobytes() == ref_inv.tobytes(), f"call {rep}: inventory differs from the oracle"
