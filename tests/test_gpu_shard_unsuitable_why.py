"""GPU suite: why each node is unsuitable on a sharded world (dra_unsuitable_why_batch_global_device, spec §17 "Sharded
form").  World contexts of this process on ONE device, wired with dra_comm_init_local / dra_peer_import_local like
test_gpu_shard_pod_capacity.py.  Every rank's four outputs must be byte for byte the oracle's answer (tests/why_oracle.py)
on the world's state: the inventory each rank holds for its own node range."""
import os
import subprocess
import sys

import numpy as np
import pytest

import shard_world as S
import why_oracle as Y
from oracle import oracle as O
from test_pod_capacity import R, _flat, problem

pytestmark = pytest.mark.gpu
SENTINEL = 0x5C
ALL = (True, True, True)
EXH = 0x4                                                # DRA_F_EXHAUSTIVE
WANTS = [ALL, (False, True, False), (True, False, True), (False, False, False), (False, False, True)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


WHY_NAMES = ("pair_why", "pair_claim", "pod_why", "claim_blocks")
WHY_N = 9                                                # DRA_WHY_N


def _world(pkg, gpus, node_off, table, world, bounds, invs=None, max_pairs=1 << 16, n_out=64, export=True, **kw):
    """rank r serving [bounds[r], bounds[r+1]) of the inventory it was given; max_pairs None: exported without room for
    the call.  shard_world.World is built without its export; dra_set_shard_why and the export and import follow here,
    as World makes them for its own size keywords."""
    W = S.World(pkg, table, node_off, gpus if invs is None else invs, world, bounds, n_out_max=n_out, export=False, **kw)
    for c in W.ctxs:
        if max_pairs is not None:
            c.set_shard_why(max_pairs)
        if world > 1 and export:
            c.shard_export(n_out, 0, want_handle=False)
    if world > 1 and export:
        for c in W.ctxs:
            c.peer_import_local(W.ctxs)
    return W


def _why(W, claims, pod_off, cands=None, flags=0, want=(True, True, True), sentinel=SENTINEL, expect=0):
    """dra_unsuitable_why_batch_global_device on every rank: every rank's four outputs (pod_why as [n_pod, WHY_N]), the
    optional ones None unless `want`.  Nothing may be written past an output, nor into one not asked for.  With `expect`
    (a failing call): every rank's whole output buffers, sentinel padding included."""
    n_pod = len(pod_off) - 1
    cn, co = (None, None) if cands is None else cands
    n_pair = n_pod * W.n_node if co is None else int(co[-1])
    keep = [S.dev(claims), S.dev(pod_off)] + ([None, None] if cn is None else [S.dev(cn), S.dev(co)])
    sizes = [n_pair, n_pair * 4, n_pod * WHY_N * 4, len(claims) * 4]
    asked = [True] + list(want)
    outs = W.outputs(sizes, sentinel)
    W.each(lambda r, c: c.unsuitable_why_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), n_pod,
                                                       S.ptr(keep[2]), S.ptr(keep[3]), n_pair,
                                                       *[t.data_ptr() if a else None for t, a in zip(outs[r], asked)],
                                                       flags=flags), expect)
    if expect:
        return [[t.cpu().numpy() for t in o] for o in outs]
    res = W.read(outs, sizes, [np.uint8, np.uint32, np.uint32, np.uint32], WHY_NAMES, asked, sentinel)
    for got in res:
        if got[2] is not None:
            got[2] = got[2].reshape(n_pod, WHY_N)
    return res


def _check(W, claims, pod_off, cands, flags, want, what, attrs=None, sels=None):
    cn, co = (None, None) if cands is None else cands
    ref = Y.why(W.state(), W.node_off, W.table, claims, pod_off, cn, co, Y.F_EXHAUSTIVE if flags else 0, attrs, sels)
    for r, got in enumerate(_why(W, claims, pod_off, cands, flags, want, SENTINEL)):
        S.same(got, ref, WHY_NAMES, f"{what} rank {r}")
    return ref


def _widest(node_off):
    return int(np.diff(np.asarray(node_off, np.int64)).max())


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven"),
                                        (4, "even"), (4, "empty")])
@pytest.mark.parametrize("width", [8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    """Dense and candidate forms, both flags, every optional-output choice, rows of W = 8, 16 and 32 lanes: every rank's
    outputs against the oracle on the world's state; the chain bit and the launch count."""
    A = pkg.api
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=60, seed=world * 10 + width)
    assert width // 2 < _widest(w.node_off) <= width
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, kind))
    try:
        rng = np.random.default_rng(world + width)
        n_pod = len(w.pod_off) - 1
        for i, (flags, form) in enumerate([(0, "dense"), (A.F_EXHAUSTIVE, "cands"), (0, "cands"), (A.F_EXHAUSTIVE, "dense"),
                                           (A.F_EXHAUSTIVE, "cands")]):
            cands = None if form == "dense" else S.cands(rng, n_pod, S.nn(w), 16)
            ref = _check(W, w.claims, w.pod_off, cands, flags, WANTS[i], f"w{world} {kind} {form} f{flags}")
            assert (ref[0] == Y.ST_OK).any() and (ref[0] != Y.ST_OK).any()
        c = W.ctxs[0]
        before = c._lib.dra_launch_count(c._h)
        _why(W, w.claims, w.pod_off)
        assert c._lib.dra_launch_count(c._h) - before == (4 if world > 1 else 3)   # prep, walk, (push,) merge
        assert c.last_chain() == {"unsuitable_why_shard"}
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_random_problems(pkg, world):
    """The CPU suite's generator: fragmented nodes of every width, pods of 0 to 33 claims with invalid ones, candidate
    lists with duplicates and strays, or the dense form; random ranges."""
    reasons = set()
    for seed in range(8):
        g, off, t, c, pod_off, cands = problem(600 * world + seed, n_node=9, n_run=60)
        rng = np.random.default_rng(seed)
        cuts = sorted(rng.integers(0, 10, world - 1).tolist())
        W = _world(pkg, g, off, t, world, [0] + cuts + [9])
        try:
            fc = None if cands is None else _flat(cands)
            for flags in (0, EXH):
                ref = _check(W, c, pod_off, fc, flags, WANTS[seed % len(WANTS)], f"seed {seed} f{flags}")
                reasons |= set(ref[0].tolist())
        finally:
            W.close()
    assert {Y.ST_OK, Y.ST_INVALID, Y.ST_NO_CAPACITY, Y.WHY_NO_NODE} <= reasons


def test_selectors_and_budget(pkg):
    """Selectors (a MIG claim whose selector no GPU passes is BAD_PROFILE) and a pod whose exhaustive search runs out of
    its budget (SEARCH_LIMIT at the MIG claim of level d), over two ranks whose copies are wrong outside their ranges."""
    t = R.default_table()
    g = np.zeros(8, O.GPU_DTYPE)
    g["flags"], g["node"] = 1, np.repeat([0, 1], 4)
    off = np.array([0, 4, 8], np.uint32)
    attrs = np.zeros(8, R.ATTR_DTYPE)
    attrs["index"] = np.arange(8) % 4
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_EQ, 0)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GT, 9))])
    small = int(np.flatnonzero(t[0]["size"] == 1)[0])
    c = np.zeros(33, O.CLAIM_DTYPE)
    c["kind"] = Y.KIND_MIG
    c["profile"] = small
    c[0]["mem_limit_mib"] = 1
    c[1]["mem_limit_mib"] = 2
    c[2]["mem_limit_mib"] = 5
    pod_off = np.array([0, 1, 2, 3, 33, 33], np.uint32)
    cands = _flat([[0, 1, S.NONE], [1, 1, 0], [2, 0], [0, 1, 1, 5], [1, 0]])
    other = g.copy()
    other["busy"] = 0x7F
    invs = [other.copy(), other.copy()]                  # rank r: the real node r, every slice taken on the other
    invs[0][:4], invs[1][4:] = g[:4], g[4:]
    W = _world(pkg, g, off, t, 2, [0, 1, 2], invs=invs, attrs=attrs, sels=sels)
    O.set_selectors(attrs, sels)
    try:
        assert W.state().tobytes() == g.tobytes()
        for flags in (0, EXH):
            for cd in (cands, None):
                ref = _check(W, c, pod_off, cd, flags, ALL, f"selectors f{flags}", attrs, sels)
                if cd is not None and flags:
                    assert ref[0][3] == Y.ST_BAD_PROFILE and ref[0][8] == Y.ST_SEARCH_LIMIT and ref[1][8] == 31
                    assert ref[3][31] == 3
    finally:
        O.set_selectors()
        W.close()


def test_diverged_copies(pkg):
    """Each rank holds the real world on its own range only, the empty inventory elsewhere: the sharded answer is the
    oracle's on the real world, while rank 0's dra_unsuitable_why_batch (its own copy taken for the world) is not.  No
    inventory word changes."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=60, seed=21)
    world = 3
    bounds = S.bounds(S.nn(w), world, "even")
    invs = []
    for r in range(world):
        g = w.empty.copy()
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        g[a:b] = w.gpus[a:b]
        invs.append(g)
    W = _world(pkg, w.gpus, w.node_off, w.table, world, bounds, invs=invs)
    try:
        assert W.state().tobytes() == w.gpus.tobytes()
        cands = S.cands(np.random.default_rng(4), len(w.pod_off) - 1, S.nn(w), 9)
        for flags in (0, EXH):
            for cd in (None, cands):
                ref = _check(W, w.claims, w.pod_off, cd, flags, ALL, f"diverged f{flags}")
                cn, co = (None, None) if cd is None else cd
                single = W.ctxs[0].unsuitable_why(w.claims, w.pod_off, cn, co, bool(flags))
                assert single[0].tobytes() != ref[0].tobytes(), "the workload does not expose stale copies"
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == invs[r].tobytes(), f"rank {r}'s live inventory changed"
            c.reset_inventory()
            assert c.get_inventory().tobytes() == invs[r].tobytes(), f"rank {r}'s pristine inventory changed"
    finally:
        W.close()


def test_the_real_flow_and_a_remap(pkg):
    """Pods placed by the sharded pods Allocate, then the sharded reasons with no sync: the oracle's answer on the world's
    state, and the same as dra_unsuitable_why_batch on rank 0 after the inventory sync.  Then the shard map moves node
    ranges between the ranks (every copy is whole after the sync), and the call still answers on the world's state."""
    import torch
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=50, seed=13)
    world = 3
    bounds = S.bounds(S.nn(w), world, "uneven")
    n_out = len(w.run_claims)
    W = _world(pkg, w.empty, w.node_off, w.table, world, bounds, invs=[w.empty] * world, n_out=n_out)
    try:
        d_rc, d_rpo = S.dev(w.run_claims), S.dev(w.run_pod_off)
        torch.cuda.synchronize()
        for c in W.ctxs:
            c.allocate_pods_global_device(d_rc.data_ptr(), len(w.run_claims), d_rpo.data_ptr(), len(w.run_pod_off) - 1,
                                          None, n_out, 0)
        cands = S.cands(np.random.default_rng(6), len(w.pod_off) - 1, S.nn(w), 12)
        got_all = _why(W, w.claims, w.pod_off, cands, EXH)
        state = W.state()
        assert state.tobytes() != w.empty.tobytes()
        befores = [c.get_inventory() for c in W.ctxs]
        assert any(b.tobytes() != state.tobytes() for b in befores)          # no rank holds the world before the sync
        ref = Y.why(state, w.node_off, w.table, w.claims, w.pod_off, *cands, Y.F_EXHAUSTIVE)
        for r, got in enumerate(got_all):
            S.same(got, ref, WHY_NAMES, f"real flow rank {r}")
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == befores[r].tobytes(), f"rank {r}: live inventory changed"
        W.sync_inventory()
        single = W.ctxs[0].unsuitable_why(w.claims, w.pod_off, *cands, True)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(single, got_all[0]))
        W.remap(S.bounds(S.nn(w), world, "even"), 2)
        for flags in (0, EXH):
            for cd in (None, cands):
                _check(W, w.claims, w.pod_off, cd, flags, ALL, f"after the remap f{flags}")
        for c in W.ctxs:
            c.reset_inventory()
            assert c.get_inventory().tobytes() == w.empty.tobytes(), "pristine inventory changed"
    finally:
        W.close()


def test_world_one_is_the_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=16, n_pending=80, seed=2)
    W = _world(pkg, w.gpus, w.node_off, w.table, 1, [0, S.nn(w)], export=False)
    try:
        rng = np.random.default_rng(0)
        for flags in (0, EXH):
            for cands in (None, S.cands(rng, len(w.pod_off) - 1, S.nn(w), 7)):
                cn, co = (None, None) if cands is None else cands
                single = W.ctxs[0].unsuitable_why(w.claims, w.pod_off, cn, co, bool(flags))
                S.same(_why(W, w.claims, w.pod_off, cands, flags)[0], single, WHY_NAMES, f"world 1 f{flags}")
        assert W.ctxs[0].last_chain() == {"unsuitable_why_shard"}
    finally:
        W.close()


def test_consecutive_calls_and_the_consequences(pkg):
    """Calls of growing and shrinking size, interleaved with sharded UnsuitableNodes and sharded pod capacity on the same
    world (call parity and the shared peer buffer): OK exactly where the sharded UnsuitableNodes sets the pair's bit with
    the same flags, and with DRA_F_EXHAUSTIVE exactly where the sharded pod capacity counts at least one copy."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=120, seed=31, fill=60)
    world = 4
    n_pod_max = len(w.pod_off) - 1
    n_pair_max = n_pod_max * S.nn(w)
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, "uneven"), max_pairs=n_pair_max,
               pairs=n_pair_max, capacity=n_pair_max)
    try:
        rng = np.random.default_rng(8)
        for it, n in enumerate((40, 120, 7, 90, 1, 120)):
            po = w.pod_off[: n + 1]
            claims = w.claims[: int(po[-1])]
            flags = EXH * (it % 2)
            cands = None if it % 3 == 0 else S.cands(rng, n, S.nn(w), 1 + it)
            ref = _check(W, claims, po, cands, flags, WANTS[it % len(WANTS)], f"call {it}")
            ok = ref[0] == Y.ST_OK
            for r, bits in enumerate(S.unsuitable(W, claims, po, cands, flags)):
                set_ = np.unpackbits(bits, bitorder="little")[: len(ok)].astype(bool)
                assert (set_ == ok).all(), f"call {it} rank {r}: OK differs from the sharded UnsuitableNodes bits"
            if flags:
                for r, got in enumerate(S.capacity(W, claims, po, cands, 1, flags, (False, False, False))):
                    assert ((got[0] >= 1) == ok).all(), f"call {it} rank {r}: OK differs from the sharded pod capacity"
            _check(W, claims, po, cands, flags, ALL, f"call {it} again")
    finally:
        W.close()


@pytest.mark.parametrize("kind", ["pod_off order", "pod_off span", "cand_off order", "cand_off span"])
def test_device_faults_fail_every_rank(pkg, kind):
    """A fault found on the device fails the call on every rank with none of the four outputs written, the per-claim
    counts included; the next call on the same world is right."""
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=17)
    world = 3
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        po = w.pod_off.copy()
        cn, co = S.cands(np.random.default_rng(0), len(po) - 1, S.nn(w), 4)
        if kind == "pod_off order":
            po[5] = po[6] + 1
        elif kind == "pod_off span":
            po[-1] -= 1
        elif kind == "cand_off order":
            co[3] = co[4] + 2
        else:
            co[0] = 1
        for flags in (0, EXH):
            outs = _why(W, w.claims, po, (cn, co), flags, ALL, sentinel=SENTINEL, expect=A.E_INVAL)
            for r, o in enumerate(outs):
                for name, h in zip(WHY_NAMES, o):
                    assert (h == SENTINEL).all(), f"{kind} f{flags}: rank {r} wrote {name}"
        # the next valid call on the same world matches the oracle
        _check(W, w.claims, w.pod_off, S.cands(np.random.default_rng(2), len(po) - 1, S.nn(w), 4), EXH, ALL, f"after {kind}")
    finally:
        W.close()


@pytest.mark.parametrize("world", [1, 2, 3])
def test_pods_without_candidates(pkg, world):
    """Every candidate list empty (n_pair 0, n_pod > 0): no pair is written, and every rank's pod_why rows and per-claim
    counts are 0.  The exchange still runs, and the next call on the same world is right."""
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=9, fill=40)
    n_pod = len(w.pod_off) - 1
    W = _world(pkg, w.gpus, w.node_off, w.table, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        empty = (np.zeros(0, np.uint32), np.zeros(n_pod + 1, np.uint32))
        for flags in (0, EXH):
            ref = _check(W, w.claims, w.pod_off, empty, flags, ALL, f"w{world} no candidates f{flags}")
            assert len(ref[0]) == 0 and not ref[2].any() and not ref[3].any()
            c = W.ctxs[0]
            before = c._lib.dra_launch_count(c._h)
            got = _why(W, w.claims, w.pod_off, empty, flags)
            assert c._lib.dra_launch_count(c._h) - before == (3 if world > 1 else 2)   # prep, (push,) merge
            for r, g in enumerate(got):
                assert not g[2].any() and g[2].shape == (n_pod, WHY_N) and not g[3].any(), f"rank {r}"
        cn, co = S.cands(np.random.default_rng(3), n_pod, S.nn(w), 3)
        co[1:6] = co[1]                                   # pods 1..4: no candidates
        keep_n = np.concatenate([cn[: co[1]], cn[co[1] + 12:]]).astype(np.uint32)
        co[6:] -= 12
        ref = _check(W, w.claims, w.pod_off, (keep_n, co), EXH, ALL, f"w{world} mixed")
        assert not ref[2][1:5].any() and ref[2].any()
    finally:
        W.close()


def test_host_side_errors(pkg):
    import torch
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=5)
    n_pod, n_node = len(w.pod_off) - 1, S.nn(w)
    W = _world(pkg, w.gpus, w.node_off, w.table, 2, S.bounds(n_node, 2, "even"), max_pairs=n_pod * n_node)
    try:
        c = W.ctxs[0]
        keep = [S.dev(w.claims), S.dev(w.pod_off)]
        cn, co = S.cands(np.random.default_rng(1), n_pod, n_node, 3)
        d_cn, d_co = S.dev(cn), S.dev(co)
        sentinel = torch.full((1 << 16,), SENTINEL, dtype=torch.uint8, device="cuda:0")
        o = sentinel.data_ptr()
        launches = c._lib.dra_launch_count(c._h)

        def call(n_pair=n_pod * n_node, flags=0, why=o, cands=(None, None), n=n_pod):
            with pytest.raises(A.DraError) as e:
                c.unsuitable_why_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n, *cands, n_pair,
                                               why, o, o, o, flags)
            return e.value.code

        assert call(flags=0x1) == A.E_INVAL                                   # unknown flags
        assert call(flags=A.F_FRESH_INVENTORY) == A.E_INVAL
        assert call(cands=(d_cn.data_ptr(), None), n_pair=int(co[-1])) == A.E_INVAL   # one candidate array alone
        assert call(cands=(None, d_co.data_ptr()), n_pair=int(co[-1])) == A.E_INVAL
        assert call(n_pair=n_pod * n_node + 1) == A.E_INVAL                   # dense n_pair != n_pod * n_node
        assert call(cands=(d_cn.data_ptr(), d_co.data_ptr()), n_pair=0xFFFFFFF1) == A.E_INVAL
        assert call(cands=(d_cn.data_ptr(), d_co.data_ptr()), n_pair=n_pod * n_node + 1) == A.E_INVAL   # above max_pairs
        assert call(n=(1 << 26) + 1, cands=(d_cn.data_ptr(), d_co.data_ptr()), n_pair=int(co[-1])) == A.E_INVAL
        assert call(why=None) == A.E_INVAL                                    # no pair_why with pairs to answer
        assert c._lib.dra_launch_count(c._h) == launches
        torch.cuda.synchronize()
        assert (sentinel.cpu().numpy() == SENTINEL).all(), "a refused call wrote an output"
        with pytest.raises(A.DraError) as e:
            c.set_shard_why(10)                                               # after the export
        assert e.value.code == A.E_STATE
        # no pods: OK, nothing enqueued on any rank
        for ctx in W.ctxs:
            ctx.unsuitable_why_global_device(keep[0].data_ptr(), 0, keep[1].data_ptr(), 0, None, None, 0, None)
            ctx.sync()
        assert c._lib.dra_launch_count(c._h) == launches
    finally:
        W.close()
    with A.Context(device=0) as c:                        # a slice over 4 GiB cannot be reserved
        with pytest.raises(A.DraError) as e:
            c.set_shard_why(0xFFFFFFF0)
        assert e.value.code == A.E_INVAL
        c.set_shard_why(800_000_000)
    # a bare dra_set_shard, a world with no export, one exported without dra_set_shard_why
    for kw in (dict(bare=True), dict(export=False), dict(max_pairs=None)):
        W = _world(pkg, w.gpus, w.node_off, w.table, 2, S.bounds(n_node, 2, "even"), **kw)
        try:
            with pytest.raises(A.DraError) as e:
                _why(W, w.claims, w.pod_off)
            assert e.value.code == A.E_STATE, kw
            if kw == dict(max_pairs=None):                # also with no pairs at all: nothing reserved to push into
                c = W.ctxs[0]
                launches = c._lib.dra_launch_count(c._h)
                empty = (np.zeros(0, np.uint32), np.zeros(n_pod + 1, np.uint32))
                with pytest.raises(A.DraError) as e:
                    _why(W, w.claims, w.pod_off, empty)
                assert e.value.code == A.E_STATE
                assert c._lib.dra_launch_count(c._h) == launches
        finally:
            W.close()
    with A.Context(device=0) as c:                        # no dra_set_shard
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        keep = [S.dev(w.claims), S.dev(w.pod_off)]
        with pytest.raises(A.DraError) as e:
            c.unsuitable_why_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n_pod, None, None,
                                           n_pod * n_node, keep[0].data_ptr())
        assert e.value.code == A.E_STATE
    # a peer set up for a different max_pairs is refused at the import
    ctxs = [A.Context(device=0) for _ in range(2)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, 2)
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
            c.set_shard_map(S.bounds(n_node, 2, "even"))
            c.set_shard_why(100 * (r + 1))
            c.shard_export(64, 0, want_handle=False)
        with pytest.raises(A.DraError) as e:
            ctxs[0].peer_import_local(ctxs)
        assert e.value.code == A.E_INVAL
    finally:
        for c in ctxs:
            c.close()


def test_multi_process():
    """tests/multi_gpu_shard_why_check.py under torchrun, one process per GPU with IPC-mapped peer buffers."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_multi_rank import _free_port
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={min(n, 4)}",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                        os.path.join(ROOT, "tests", "multi_gpu_shard_why_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
