"""The sharded Allocate's problems at the record limits — TEST INFRASTRUCTURE ONLY, needs no GPU.

tests/test_gpu_shard_limits.py runs these through dra_allocate_batch_global_device and tests/test_shard_limit_problems.py
checks on the CPU that they reach what the GPU file relies on.  Everything is built here once, so both files see the same
seeds, splits and paddings:
  form a     tests/limit_problems.py's problems on worlds of 1-4 contexts: world 2 at every split point, worlds 3 and 4
             at the even, uneven and empty bounds and one map whose last rank holds exactly one non-empty node
  form b     a problem behind one empty node 0, on the world-1 shard [1, n_node), padded with claims naming node 0 (which
             the shard drops) and interleaved with them so that kept claims straddle the compaction's tile boundaries
  selectors  synth.mixed problems with synth.with_selectors' table, or with seeded random selector programs
  packets    one-node fixtures whose records touch the top of the packet's start, size, profile and status fields
The slot rule of k_shard_compact is restated here (`kernel_slots`) so that the CPU file can check it against
records.claim_slots."""
from __future__ import annotations

import importlib
from types import SimpleNamespace

import numpy as np

import limit_problems as LP
from preempt_problems import _Rng
from test_gpu_limits import FIXTURES, SEEDS, _fixture, _tile
from shard_world import bounds as _bounds
from test_oracle_selector_properties import selector_programs

PKG = importlib.import_module("k8s-dra-driver_b200")
R = PKG.records
NONE = 0xFFFFFFFF
SMALL_TILE, LARGE_TILE = 256, 2048          # the compaction's tiles: 256 claims up to 262,144 claims, 2,048 beyond


def as_workload(pb, **extra):
    """An LP.Problem with the attributes the sharded helpers of test_gpu_shard.py read."""
    return SimpleNamespace(gpus=pb.gpus, node_off=pb.node_off, table=pb.table, claims=pb.claims, out_off=pb.out_off,
                           n_out=int(pb.n_out), n_node=len(pb.node_off) - 1, n_claim=len(pb.claims), n_gpu=len(pb.gpus),
                           **extra)


def problems():
    """test_gpu_limits.py's problems (its seeds, DRA_PROP_EXAMPLES honoured), then its five fixtures."""
    return [as_workload(pb, name=f"seed {s}") for s, pb in ((s, LP.random_problem(s)) for s in SEEDS) if len(pb.claims)] + \
        [as_workload(_fixture(n), name=n) for n in FIXTURES]


# ---- form a: worlds of contexts on one device ------------------------------------------------------------------------
def last_rank_map(w, world):
    """Bounds whose last rank holds exactly one non-empty node (the last one); the other ranks split the rest evenly."""
    width = np.diff(w.node_off.astype(np.int64))
    full = np.nonzero(width)[0]
    j = int(full[-1]) if len(full) else w.n_node - 1
    return [j * r // (world - 1) for r in range(world)] + [w.n_node]


def splits(w):
    """(world, bounds, stray_rank) of form a: world 1, world 2 at every split point with the strays on rank 0 and then 1,
    worlds 3 and 4 at the even, uneven and empty bounds and at the last-rank map."""
    n = w.n_node
    out = [(1, [0, n], 0)]
    out += [(2, [0, s, n], stray) for s in range(n + 1) for stray in (0, 1)]
    for world in (3, 4):
        out += [(world, _bounds(n, world, kind), stray) for kind, stray in (("even", 0), ("uneven", world - 1), ("empty", 1))]
        out.append((world, last_rank_map(w, world), 0))
    return out


def kernel_slots(claims, n_node, have_off):
    """OutRec slots per claim as k_shard_compact counts them: `count` for a well-formed GPU claim that names a node (with
    out_off, or count 1 without it), else one."""
    kind, cnt, node = claims["kind"], claims["count"].astype(np.int64), claims["node"].astype(np.int64)
    ok = (kind == R.KIND_GPU) & (node < n_node) & (cnt >= 1) & (cnt <= R.MAX_COUNT) & (bool(have_off) | (cnt == 1))
    return np.where(ok, cnt, 1)


def owner(claims, n_node, bounds, stray_rank):
    """The rank that answers each claim: the one whose node range holds its node, stray_rank for claims naming no node."""
    node = claims["node"].astype(np.int64)
    o = np.searchsorted(np.asarray(bounds[1:-1], np.int64), node, side="right")
    return np.where(node >= n_node, stray_rank, o)


def slot_form(w, form):
    """(out_off, n_out) of a slot form: "off" the batch's own out_off, "nooff" none, one slot per claim."""
    return (w.out_off, w.n_out) if form == "off" else (None, w.n_claim)


# ---- form b: one world-1 sub-range shard, padded past each compaction and chain limit ---------------------------------
def behind_empty_node(w):
    """w between an empty node 0 and a node of 4 GPUs at the end (the shard [1, n_node - 1) leaves both out): its nodes
    and its claims' nodes shift up by one, claims naming no node still name none; its GPU indices do not change."""
    n = w.n_node
    tail, _ = R.make_inventory([4], mig=True)
    tail["model"] = int(np.nonzero(w.table["start_mask"].any(axis=1))[0][0])
    tail["node"] = n + 1
    g = np.concatenate([w.gpus, tail])
    g["node"][: w.n_gpu] += 1
    off = np.concatenate([[0], w.node_off, [w.node_off[-1] + 4]]).astype(np.uint32)
    c = w.claims.copy()
    node = c["node"].astype(np.int64)
    c["node"] = np.where(node == NONE, NONE, np.where(node < n, node + 1, node + 2)).astype(np.uint32)
    oo, n_out = R.out_offsets(c, n + 2)
    extra = {}
    if getattr(w, "attrs", None) is not None:
        extra["attrs"] = np.concatenate([w.attrs, np.zeros(4, w.attrs.dtype)])
    return SimpleNamespace(**{**vars(w), "gpus": g, "node_off": off, "claims": c, "out_off": oo, "n_out": int(n_out),
                              "n_node": n + 2, "n_gpu": len(g), "lo": 1, "hi": n + 1, **extra})


def _pad(n):
    """n claims that the shard drops: 1-slice MIG claims naming node 0 and the last node in turn."""
    c = np.zeros(n, R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_MIG, 1
    return c


def place(n, n_total, tile):
    """Positions of n claims in a batch of n_total: the claims cut in order into chunks, one chunk around each chosen tile
    boundary (evenly spread, all of them when there are claims enough), half of it before and half from the boundary on,
    with one dropped claim between neighbours."""
    bounds = np.arange(tile, n_total - tile // 2, tile, dtype=np.int64)     # (room for half a tile after the last)
    m = max(1, min(len(bounds), n // 2))
    bounds = bounds[np.round(np.linspace(0, len(bounds) - 1, m)).astype(np.int64)]
    pos = []
    for b, chunk in zip(bounds, np.array_split(np.arange(n), m)):
        s = len(chunk)
        pos += [int(b) - 2 * (s // 2) + 2 * t for t in range(s)]
    pos = np.array(pos, np.int64)
    assert (np.diff(pos) > 0).all() and pos[0] >= 0 and pos[-1] < n_total
    return pos


def SORT_CHAIN_PAD(w):
    """The batch of the one-CTA counting sort's test: at most 8,192 claims, chunks of at most a quarter tile"""
    return 4 * w.n_claim + 600


def padded(w, n_total):
    """behind_empty_node(w) padded to n_total claims that the shard drops (_pad), its own
    claims placed by `place` at the compaction's tile (256 up to 262,144 claims, else 2,048).  `pos`: where they went."""
    v = behind_empty_node(w)
    tile = SMALL_TILE if n_total <= 256 * 1024 else LARGE_TILE
    pos = place(v.n_claim, n_total, tile)
    c = _pad(n_total)
    c["node"] = np.where(np.arange(n_total) % 2, v.n_node - 1, 0)
    c[pos] = v.claims
    oo, n_out = R.out_offsets(c, v.n_node)
    return SimpleNamespace(**{**vars(v), "claims": c, "out_off": oo, "n_out": int(n_out), "n_claim": n_total, "pos": pos,
                              "tile": tile})


def tiled(w, min_nodes):
    """w repeated over at least min_nodes nodes (test_gpu_limits._tile) by behind_empty_node, with a few dropped claims."""
    pb = _tile(LP.Problem(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out), min_nodes)
    v = behind_empty_node(as_workload(pb, name=f"{w.name} tiled"))
    n = v.n_claim                                        # a dropped claim before every 4,096 of them
    pos = np.arange(n) + np.arange(n) // 4096 + 1
    c = _pad(n + n // 4096 + 1)
    c["node"] = v.n_node - 1
    c[pos] = v.claims
    oo, n_out = R.out_offsets(c, v.n_node)
    return SimpleNamespace(**{**vars(v), "claims": c, "out_off": oo, "n_out": int(n_out), "n_claim": len(c), "pos": pos})


# ---- selectors -------------------------------------------------------------------------------------------------------
SEL_SEEDS = list(range(8))


def selector_problem(seed):
    """synth.mixed with synth.with_selectors' table (even seeds) or with random programs of
    test_oracle_selector_properties.selector_programs drawn from the seed (odd seeds), carried by every 1st-4th claim.
    One GPU claim of count 3 on the last node names the id just beyond the table."""
    w = PKG.synth.mixed(700, 15, 400 + seed, invalid=True)
    c = w.claims
    if seed % 2 == 0:
        attrs, sels = PKG.synth.with_selectors(w, seed=seed)
    else:
        attrs, sels, sid = selector_programs(_Rng(np.random.default_rng(seed)), w.n_gpu)
        pick = (np.arange(w.n_claim) % (seed % 4 + 1)) == 0
        gm = pick & ((c["kind"] == R.KIND_GPU) | (c["kind"] == R.KIND_MIG))
        c["mem_limit_mib"] = np.where(gm, sid, c["mem_limit_mib"])
        c["group"] = np.where(pick & (c["kind"] == R.KIND_SHARED), sid, c["group"])
    beyond = 100 + seed
    c[beyond] = (R.KIND_GPU, 0, 3, w.n_node - 1, len(sels) + 1, 0)
    w.out_off, w.n_out = R.out_offsets(c, w.n_node)
    return SimpleNamespace(gpus=w.gpus, node_off=w.node_off, table=w.table, claims=c, out_off=w.out_off, n_out=int(w.n_out),
                           n_node=w.n_node, n_claim=w.n_claim, n_gpu=w.n_gpu, attrs=attrs, sels=sels, beyond=beyond,
                           name=f"selectors {seed}")


def selector_splits(w):
    """Form a for the selector problems: world 1, world 2 at the middle with the strays on rank 1, worlds 3 and 4 even and
    uneven.  The claim beyond the table sits on the last node, so never on the stray rank's nodes at world > 1."""
    n = w.n_node
    return [(1, [0, n], 0), (2, [0, n // 2, n], 0), (3, _bounds(n, 3, "even"), 0), (4, _bounds(n, 4, "uneven"), 0),
            (4, _bounds(n, 4, "empty"), 1)]


# ---- packet-format fixtures: one node, on the last rank ----------------------------------------------------------------
PACKET_FIXTURES = ["start15", "size16", "gpu32", "profile_bytes", "statuses"]


def packet_fixture(name):
    """One node (of 32 GPUs) and claims whose OutRecs touch the top of their packet fields; claims naming no node too."""
    U32 = LP.U32
    MIG, GPU, SH = R.KIND_MIG, R.KIND_GPU, R.KIND_SHARED
    t = R.empty_table()
    t[3, 0] = (1, 0, 0x8000)                             # 1 slice at start 15 only
    t[3, 1] = (16, 0, 0x0001)                            # the whole 16-slice GPU
    t[3, 2] = (4, 0, 0x1111)                             # 4 slices at 0, 4, 8, 12
    t[3, 3] = (0, 0, 0)                                  # unoffered
    g, off = R.make_inventory([32], mig=True)
    g["model"] = 3
    rows = []
    stray = [(MIG, 15, 1, NONE, 0), (GPU, 0, 33, 1, 0), (SH, 0, 1, 8, 0)]      # (kind, profile, count, node, mem / sel)
    if name == "start15":
        rows = [(MIG, 0, 1, 0, 0)] * 40                  # 32 at start 15, then NO_CAPACITY
    elif name == "size16":
        rows = [(MIG, 1, 1, 0, 0)] * 33
    elif name == "gpu32":
        g["flags"] = 0
        rows = [(GPU, 0, 32, 0, 0), (GPU, 0, 33, 0, 0), (GPU, 0, 0, 0, 0), (GPU, 0, 1, 0, 0)]
    elif name == "profile_bytes":
        rows = [(MIG, 0x0F, 1, 0, 0), (MIG, 0xFF, 1, 0, 0), (3, 0xFF, 1, 0, 0), (255, 0x0F, 1, 0, 0), (MIG, 0x10, 1, 0, 0)]
    elif name == "statuses":
        # GPUs 0-15 take 64 4-slice instances (slices 12-15 end up busy), GPUs 16-31 serve shared claims of 1000 MiB
        g["flags"][16:] = 0
        g["mem_free_mib"][16:] = 1000
        rows = [(MIG, 2, 1, 0, 0)] * 65 + [(MIG, 3, 1, 0, 0)] + [(MIG, 0, 1, 0, 0)] * 2 + \
               [(SH, 0, 1, 0, 2000), (SH, 0, 1, 0, 1000), (SH, 0, 1, 0, U32)]
    else:
        raise KeyError(name)
    rows = rows + stray
    c = np.zeros(len(rows), R.CLAIM_DTYPE)
    for i, (kind, prof, cnt, node, x) in enumerate(rows):
        c[i] = (kind, prof, cnt, node, x, 0)
    if name == "statuses":                               # a co-location run of two 1-slice claims: no room left
        c["group"][66:68] = 7
    oo, n_out = R.out_offsets(c, 1)
    return SimpleNamespace(gpus=g, node_off=off, table=t, claims=c, out_off=oo, n_out=int(n_out), n_node=1,
                           n_claim=len(c), n_gpu=len(g), name=name)


PACKET_EXPECT = {   # what each fixture's OutRecs must hold (on the oracle, before the device runs)
    "start15": lambda o: ((o["start"] == 15) == (o["status"] == R.ST_OK)).all() and (o["status"] == R.ST_OK).sum() == 32,
    "size16": lambda o: ((o["size"] == 16) == (o["status"] == R.ST_OK)).all() and (o["status"] == R.ST_OK).sum() == 32,
    "gpu32": lambda o: (o["status"][:32] == R.ST_OK).all() and (o["status"][32:34] == R.ST_INVALID).all(),
    "profile_bytes": lambda o: {0x0F, 0xFF} <= set(o["profile"][o["status"] == R.ST_INVALID].tolist()),
    "statuses": lambda o: set(range(6)) <= set(o["status"].tolist()),
}
