"""GPU suite: every Allocate kernel chain at its dispatch boundaries, bit-exact with the oracle.

The library picks one of about a dozen kernel chains from the claim count, the node count and the device's SM count.  Each
row of the table below is a shape on one side of one threshold and the chain that shape must take: the test asks the library
which kernels it enqueued (dra_debug_last_chain) instead of re-deriving the dispatch, so a threshold that moves fails here
loudly rather than silently moving coverage elsewhere.  Shapes are built from the SM count (`S`), so the table holds on any
H100.  Every row runs synth.mixed (invalid claims, counts > 1, co-location groups); rows about a counter or a chain limit
also run skewed forms of the same shape:
  hot        one node takes >= 90 % of the claims, and every claim of the first 65,536 (whole hist tiles on one node)
  nonode     every claim names no node (n_node, n_node + 1000, 0xFFFFFFFF)
  empty_ends nodes 0 and n_node - 1 have no GPU, and every fourth claim names one of them
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SORT8 = {"hist8", "scan8", "scatter"}              # CTA-wide histogram, 2048-claim tiles, one warp per node in the scan
WARP = {"hist_warp", "scan", "scatter"}            # one-warp histogram tiles (node ranges too wide for the CTA-wide form)
D4 = ("mixed", "hot", "nonode", "empty_ends")
STAGED_CAP = 11_117                                # most claims whose staged layout fits the single-launch kernel's shared memory

# id, context flags, shape(S) -> (n_claim, n_node), chain, hist tile (0: no histogram kernel), distributions
ROWS = [
    # single-launch kernel: claim array staged in shared memory or streamed
    ("staged_max", "nodirect", lambda S: (STAGED_CAP, S - 1), {"fused_staged"}, 0, D4),
    ("stream_min", "nodirect", lambda S: (STAGED_CAP + 1, S - 1), {"fused_stream"}, 0, D4),
    # fused vs sort, one wave of CTAs (n_node + 1 <= S): 14,000 claims
    ("one_wave_fused_max", "nodirect", lambda S: (14_000, S - 1), {"fused_stream"}, 0, D4),
    ("one_wave_sort_min", "nodirect", lambda S: (14_001, S - 1), SORT8 | {"pack1"}, 2048, D4),
    # fused vs sort, two waves: 7,500 claims
    ("one_wave_10k", "nodirect", lambda S: (10_000, S - 1), {"fused_staged"}, 0, ("mixed",)),
    ("two_waves_10k", "nodirect", lambda S: (10_000, S), SORT8 | {"pack1"}, 2048, ("mixed",)),
    ("two_waves_fused_max", "nodirect", lambda S: (7_500, S), {"fused_staged"}, 0, D4),
    ("two_waves_sort_min", "nodirect", lambda S: (7_501, S), {"bucket_small", "pack1"}, 0, D4),
    # n_node * n_claim: 3,000,000 fused, 3,000,001 = 853 x 3,517 not
    ("work_cap", "nodirect", lambda S: (3_000, 1_000), {"fused_staged"}, 0, D4),
    ("work_cap_plus_1", "nodirect", lambda S: (3_517, 853), {"bucket_small", "pack1"}, 0, D4),
    # node cap of the single-launch kernel (many waves of CTAs); one past it takes the one-warp histogram
    ("fused_nodes_max", "nodirect", lambda S: (150, 16_384), {"fused_staged"}, 0, D4),
    ("fused_nodes_over", "nodirect", lambda S: (150, 16_385), WARP | {"pack4"}, 256, D4),
    # the one-CTA counting sort: 8,192 claims, and its shared memory at 8,192 claims (2,769 nodes)
    ("bucket_small_claims_max", 0, lambda S: (8_192, S), {"bucket_small", "pack1"}, 0, D4),
    ("hist8_claims_min", 0, lambda S: (8_193, S), SORT8 | {"pack1"}, 2048, D4),
    ("bucket_small_smem_max", 0, lambda S: (8_192, 2_769), {"bucket_small", "pack4"}, 0, D4),
    ("bucket_small_smem_over", 0, lambda S: (8_192, 2_770), SORT8 | {"pack4"}, 2048, D4),
    # CTA-wide histogram: 2048-claim tiles up to S tiles, then tiles grown to a multiple of 2048 (cap 32,768: u16 ranks)
    ("hist8_tile_fixed_max", 0, lambda S: (S * 2048, 1_000), SORT8 | {"pack1"}, 2048, D4),
    ("hist8_tile_grown_min", 0, lambda S: (S * 2048 + 1, 1_000), {"hist8_multi", "scan8", "scatter", "pack1"}, 4096, D4),
    ("hist8_tile_cap", 0, lambda S: (max(4_500_000, S * 32_768 + 100_000), 1_000),
     {"hist8_multi", "scan8", "scatter", "pack1"}, 32_768, ("mixed", "hot")),
    # the scan of the tile histograms: one warp per node up to 524,288 counters, coalesced rows beyond
    ("scan8_max", 0, lambda S: (S * 2048, 524_288 // S - 1), SORT8 | {"pack4"}, 2048, D4),
    ("scan_rows_min", 0, lambda S: (S * 2048, 524_288 // S), {"hist8", "scan_rows", "scatter", "pack4"}, 2048, D4),
    # one warp per node while 16 warps per SM cover the nodes, then CTAs of four warps walking nodes
    ("pack1_max", 0, lambda S: (20_000, 16 * S), SORT8 | {"pack1"}, 2048, D4),
    ("pack4_min", 0, lambda S: (20_000, 16 * S + 1), SORT8 | {"pack4"}, 2048, D4),
    # CTA-wide histogram while 8 x (n_node + 2) u16 counters fit 200 KiB, one-warp tiles beyond (cap 65,504: u16 counters)
    ("hist8_nodes_max", 0, lambda S: (50_000, 12_798), SORT8 | {"pack4"}, 2048, D4),
    ("hist_warp_nodes_min", 0, lambda S: (50_000, 12_799), WARP | {"pack4"}, 800, D4),
    ("hist_warp_tile_cap", 0, lambda S: (4_300_000, 13_000), WARP | {"pack4"}, 65_504, ("mixed", "hot")),
    # node limit of the bucketing: (n_node + 1) u16 counters in 200 KiB
    ("bucketing_nodes_max", 0, lambda S: (5_000, 102_399), WARP | {"pack4"}, 256, ("mixed", "nonode")),
    # (large batches with wave-sized tiles, the row-wise scan of a big matrix: test_gpu_parity.py, test_large_batches_match_oracle)
]
CASES = [pytest.param(r, d, id=f"{r[0]}-{d}") for r in ROWS for d in r[5]]


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _flags(pkg, name):
    return {0: 0, "nodirect": pkg.api.CFG_NO_DIRECT, "resident": pkg.api.CFG_RESIDENT}[name]


def workload(pkg, n_claim, n_node, dist, seed=11):
    """synth.mixed at this shape, then the skew of `dist` (claims' slots recomputed after any node change)."""
    R = pkg.records
    w = pkg.synth.mixed(n_claim, n_node, seed, invalid=True)
    c, i = w.claims, np.arange(n_claim)
    if dist == "hot":
        hot = 1 if n_node > 2 else 0                      # (mixed gives node 1 eight GPUs)
        m = i % 10 != 0
        m[:65_536] = True
        c["node"][m] = hot
    elif dist == "nonode":
        c["node"] = np.where(i % 3 == 0, n_node, np.where(i % 3 == 1, n_node + 1000, 0xFFFFFFFF)).astype(np.uint32)
    elif dist == "empty_ends":
        last = int(w.node_off[-2])                        # drop the last node's GPUs (mixed already leaves node 0 empty)
        w.gpus = w.gpus[:last].copy()
        w.node_off = w.node_off.copy()
        w.node_off[-1] = last
        assert w.node_off[1] == 0
        c["node"] = np.where(i % 8 == 0, 0, np.where(i % 8 == 4, n_node - 1, c["node"])).astype(np.uint32)
    else:
        assert dist == "mixed"
    w.out_off, w.n_out = R.out_offsets(c, n_node)
    return w


def assert_same(out, inv, ref_out, ref_inv, what=""):
    if out.tobytes() != ref_out.tobytes():
        bad = np.nonzero(out.view(np.uint64) != ref_out.view(np.uint64))[0]
        raise AssertionError(f"{what}: {len(bad)} OutRecs differ, first at {bad[0]}: cuda={out[bad[0]]} oracle={ref_out[bad[0]]}")
    if inv.tobytes() != ref_inv.tobytes():
        bad = np.nonzero(inv.view("V16") != ref_inv.view("V16"))[0]
        raise AssertionError(f"{what}: inventory differs at gpu {bad[0]}: cuda={inv[bad[0]]} oracle={ref_inv[bad[0]]}")


@pytest.mark.parametrize("row,dist", CASES)
def test_chain_at_boundary(pkg, oracle, row, dist):
    name, cfg, shape, chain, tile, _ = row
    S = _sms()
    n_claim, n_node = shape(S)
    w = workload(pkg, n_claim, n_node, dist)
    with pkg.api.Context(device=0, flags=_flags(pkg, cfg)) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        out = c.allocate(w.claims, w.out_off, w.n_out)
        inv = c.get_inventory()
        got_chain, got_tile = c.last_chain(), c.last_hist_tile()
    ref_out, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out, threads=8)
    assert_same(out, inv, ref_out, ref_inv, f"{name} {dist}: {n_claim} claims x {n_node} nodes, {S} SMs")
    assert got_chain == chain, f"{name}: {n_claim} x {n_node} on {S} SMs took {sorted(got_chain)}"
    assert got_tile == tile, f"{name}: hist tile {got_tile}"


def test_bucketing_node_limit_is_an_error(pkg):
    """One node past the bucketing limit: DRA_E_INVAL before any kernel runs, the inventory untouched, the context usable."""
    w = workload(pkg, 5_000, 102_400, "mixed")
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        with pytest.raises(pkg.api.DraError) as e:
            c.allocate(w.claims, w.out_off, w.n_out)
        assert e.value.code == pkg.api.E_INVAL
        assert c.get_inventory().tobytes() == w.gpus.tobytes()
        small = workload(pkg, 2_000, 50, "mixed")
        c.set_inventory(small.gpus, small.node_off)
        c.allocate(small.claims, small.out_off, small.n_out)


def _slots_exactly(pkg, w, target):
    """Raise the counts of valid GPU claims (up to 32) until the batch has exactly `target` OutRec slots."""
    R = pkg.records
    c = w.claims
    need = target - int(R.claim_slots(c, w.n_node).sum())
    for i in np.nonzero((c["kind"] == R.KIND_GPU) & (c["node"] < w.n_node) & (c["count"] >= 1) & (c["count"] <= 32))[0]:
        if need <= 0:
            break
        add = min(need, 32 - int(c["count"][i]))
        c["count"][i] += add
        need -= add
    assert need == 0
    w.out_off, w.n_out = R.out_offsets(c, w.n_node)
    assert w.n_out == target
    return w


@pytest.mark.parametrize("n_claim,n_out,served", [
    (STAGED_CAP, None, True), (STAGED_CAP + 1, None, False),
    (STAGED_CAP, 2 * STAGED_CAP, True), (STAGED_CAP, 2 * STAGED_CAP + 1, False)])
def test_resident_capacity(pkg, oracle, n_claim, n_out, served):
    """DRA_CFG_RESIDENT serves batches up to the staged capacity in claims and twice that in OutRecs; one more of either
    stops the resident kernel and takes the launched path."""
    A, R = pkg.api, pkg.records
    S = _sms()
    w = workload(pkg, n_claim, S - 1, "mixed", seed=21)
    if n_out is not None:
        _slots_exactly(pkg, w, n_out)
    ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out, threads=8)
    with A.Context(device=0, flags=A.CFG_RESIDENT) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        pc = A.PinnedBuffer(w.n_claim, R.CLAIM_DTYPE); pc.array[:] = w.claims
        pf = A.PinnedBuffer(w.n_claim, np.uint32); pf.array[:] = w.out_off
        po = A.PinnedBuffer(w.n_out, R.OUT_DTYPE); po.array[:] = 0
        b0 = c.serve_batches()
        got = c.allocate(pc.array, pf.array, w.n_out, out=po.array).copy()
        chain, batches = c.last_chain(), c.serve_batches() - b0
        inv = c.get_inventory()
        for p in (pc, pf, po):
            p.free()
    assert_same(got, inv, ref, ref_inv, f"resident {n_claim} claims, {w.n_out} slots")
    if served:
        assert chain == {"serve"} and batches == 1
    else:
        assert batches == 0 and chain == ({"fused_direct"} if n_claim <= STAGED_CAP else {"fused_stream"}), chain


@pytest.mark.parametrize("n_claim,chain", [(STAGED_CAP, {"fused_direct"}), (STAGED_CAP + 1, {"fused_stream"})])
def test_direct_io_capacity(pkg, oracle, n_claim, chain):
    """A default context lets the single-launch kernel read and write the pinned host buffers itself while the claim
    array stages in shared memory; one claim more and the batch goes through copy-engine transfers."""
    S = _sms()
    w = workload(pkg, n_claim, S - 1, "mixed", seed=22)
    with pkg.api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        out = c.allocate(w.claims, w.out_off, w.n_out)
        inv = c.get_inventory()
        got = c.last_chain()
    ref, ref_inv = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out, threads=8)
    assert_same(out, inv, ref, ref_inv, f"direct I/O {n_claim} claims")
    assert got == chain
