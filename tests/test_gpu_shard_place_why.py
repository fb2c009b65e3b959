"""GPU suite: why place pods put each pod where it did across a sharded world (dra_place_pods_why_batch_global_device,
spec §18 "Sharded form").  World contexts of this process on ONE device (tests/shard_world.World).  Every rank's four
reason outputs must be byte for byte the oracle's (tests/place_why_oracle.py) on the world's state, and the table,
pod_node and every rank's own GPU range byte for byte what dra_place_pods_batch_global_device leaves: asking for reasons
changes no placement."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from test_gpu_shard_place import _flags, _forms
from test_place_pods import NONE, _flat, placed_offsets

import place_oracle as P
import place_why_oracle as PW
import shard_world as S
import why_oracle as Y
from oracle import oracle as O

pytestmark = pytest.mark.gpu
SENTINEL = 0x5C
N_OUT_MAX = 1 << 16
WHY_N = 9                                                # DRA_WHY_N
NAMES = ("pod_node", "pair_why", "pair_claim", "pod_why", "claim_blocks")
WANTS = [(True, True, True), (False, True, False), (True, False, True), (False, False, False)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _world(pkg, w, world, bounds, stray_rank=0, max_pods=4096, max_pairs=1 << 16, attrs=None, sels=None, cap_per_rank=0,
           invs=None):
    """rank r serving [bounds[r], bounds[r+1]); room for the replicated pod states (max_pods) and, unless max_pairs is None,
    the reasons' exchange (max_pairs), both reserved before the export"""
    W = S.World(pkg, w.table, w.node_off, w.gpus if invs is None else invs, world, bounds, stray_rank, attrs, sels,
                export=False, n_out_max=N_OUT_MAX, cap_per_rank=cap_per_rank, place=max_pods)
    for c in W.ctxs:
        if max_pairs is not None:
            c.set_shard_why(max_pairs)
        if world > 1:
            c.shard_export(N_OUT_MAX, cap_per_rank, want_handle=False)
    if world > 1:
        for c in W.ctxs:
            c.peer_import_local(W.ctxs)
    return W


def _why(W, claims, pod_off, cands, out_off, n_out, flags=0, want=(True, True, True), expect=0):
    """dra_place_pods_why_batch_global_device on every rank: every rank's (table, [pod_node, pair_why, pair_claim,
    pod_why as [n_pod, WHY_N], claim_blocks]), the optional outputs None unless `want`.  Nothing may be written past an
    output, nor into one not asked for.  With `expect` (a failing call): every rank's whole output buffers."""
    cn, co = (None, None) if cands is None else cands
    n_pod = len(pod_off) - 1
    n_pair = 0 if co is None else int(co[-1])
    n_why = n_pod * W.n_node if co is None else n_pair
    keep = [S.dev(claims), S.dev(pod_off), None if out_off is None else S.dev(out_off)] + \
        ([None, None] if co is None else [S.dev(cn), S.dev(co)])
    sizes = [n_pod * 4, n_why, n_why * 4, n_pod * WHY_N * 4, len(claims) * 4]
    asked = [True, True] + list(want)
    outs = W.outputs(sizes, SENTINEL)
    W.each(lambda r, c: c.place_pods_why_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), n_pod,
                                                       S.ptr(keep[3]), S.ptr(keep[4]), n_pair, S.ptr(keep[2]), n_out,
                                                       *[t.data_ptr() if a else None for t, a in zip(outs[r], asked)],
                                                       flags=flags), expect)
    if expect:
        return [[t.cpu().numpy() for t in o] for o in outs]
    res = W.read(outs, sizes, [np.uint32, np.uint8, np.uint32, np.uint32, np.uint32], NAMES, asked, SENTINEL)
    for got in res:
        if got[3] is not None:
            got[3] = got[3].reshape(n_pod, WHY_N)
    return [(c.gather_read(np.zeros(n_out, dtype=W.pkg.records.OUT_DTYPE)), got) for c, got in zip(W.ctxs, res)]


def _check(W, w, claims, pod_off, cn, co, out_off, n_out, flags, what, want=(True, True, True), attrs=None, sels=None):
    """One call against the §18 oracle on the world's state: every rank's table, pod_node and reasons, its own range the
    oracle's and nothing written outside it, pod_node the node of the pod's first OK pair, the chain taken.  With
    DRA_F_FRESH_INVENTORY the same call without reasons follows from the same start state, and must place alike."""
    api = W.pkg.api
    before = W.inventories()
    src = w.gpus if flags & api.F_FRESH_INVENTORY else W.state()
    ref = PW.place_why(src, w.node_off, w.table, claims, pod_off, cn, co, out_off, n_out, flags & Y.F_EXHAUSTIVE, attrs,
                       sels)
    res = _why(W, claims, pod_off, None if co is None else (cn, co), out_off, n_out, flags, want)
    for r, (table, got) in enumerate(res):
        assert table.tobytes() == ref[0].tobytes(), f"{what}: rank {r} table"
        S.same(got, [ref[1]] + list(ref[3:]), NAMES, f"{what} rank {r}")
    W.assert_ranges(before, ref[2], what)
    assert W.ctxs[0].last_chain() >= {"place_shard", "place_why"}
    sizes = np.diff(np.asarray(pod_off, np.int64))
    for p in range(len(pod_off) - 1):                    # pod_node is the node of the pod's first OK pair
        if not 0 < sizes[p] <= 32:
            continue
        k0, k1 = (p * w.n_node, (p + 1) * w.n_node) if co is None else (int(co[p]), int(co[p + 1]))
        ok = np.flatnonzero(ref[3][k0:k1] == Y.ST_OK)
        first = NONE if not len(ok) else (int(ok[0]) if co is None else int(cn[k0 + ok[0]]))
        assert int(ref[1][p]) == first, f"{what}: pod {p}"
    if flags & api.F_FRESH_INVENTORY:
        after = W.inventories()
        plain = S.place(W, claims, pod_off, None if co is None else (cn, co), out_off, n_out, flags)
        for r, (table, node) in enumerate(plain):
            assert table.tobytes() == res[r][0].tobytes() and node.tobytes() == res[r][1][0].tobytes(), f"{what}: rank {r}"
        for r, inv in enumerate(W.inventories()):
            assert inv.tobytes() == after[r].tobytes(), f"{what}: rank {r} inventory differs from the call without reasons"
    return ref


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_matches_oracle(pkg, world):
    """Every candidate form of the sharded place-pods suite on even, uneven and empty ranges, the flag combinations one
    after the other on one world, the optional outputs in turn."""
    rng = np.random.default_rng(world)
    kind = ["even", "uneven", "empty", "uneven"][world - 1]
    w, pod_off = pkg.synth.pods(300, 14, 100 + world)
    n_pod = len(pod_off) - 1
    bounds = S.bounds(w.n_node, world, kind)
    W = _world(pkg, w, world, bounds, world - 1)
    try:
        reasons = set()
        for i, (name, (cn, co)) in enumerate(_forms(rng, n_pod, w.n_node, bounds).items()):
            flags = _flags(pkg.api)[i % 4]
            ref = _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), flags, f"{name} flags {flags}", WANTS[i % 4])
            reasons |= set(ref[3].tolist())
            if name != "duplicates":
                assert (ref[1] != NONE).any() and (ref[1] == NONE).any(), name
        assert {Y.ST_OK} < reasons
    finally:
        W.close()


@pytest.mark.parametrize("world", [1, 3])
def test_mixed_pods_and_selectors(pkg, world):
    """Pods cut from synth.mixed with selectors: empty pods, a pod of more than 32 claims, malformed claims, GPU claims of
    count > 1 (out_off), random candidates with strays across ranks."""
    api = pkg.api
    rng = np.random.default_rng(30 + world)
    w = pkg.synth.mixed(900, 13, 70 + world, invalid=True)
    attrs, sels = pkg.synth.with_selectors(w, world)
    bounds = S.bounds(w.n_node, world, "even")
    claims, pod_off, _, _ = S.malformed_mixed(pkg, w, bounds, rng, False)
    out_off, n_out = placed_offsets(pkg.records, claims, w.n_node)
    n_pod = len(pod_off) - 1
    cn = rng.integers(0, w.n_node + 2, n_pod * 5).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 5).astype(np.uint32)
    W = _world(pkg, w, world, bounds, 0, attrs=attrs, sels=sels)
    O.set_selectors(attrs, sels); P.set_selectors(attrs, sels)      # (the reasons oracle builds on both C oracles)
    try:
        seen = set()
        for flags in (0, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY):
            for c_, o_ in ((cn, co), (None, None)):
                ref = _check(W, w, claims, pod_off, c_, o_, out_off, int(n_out), flags, f"mixed flags {flags}",
                             attrs=attrs, sels=sels)
                seen |= set(ref[3].tolist())
        assert {Y.ST_OK, Y.ST_INVALID, Y.WHY_NO_NODE} <= seen
    finally:
        O.set_selectors(); P.set_selectors()
        W.close()


def test_hand_offs(pkg):
    """A pod whose failed, chosen and dry-run pairs fall on three ranks: 7 x 1g + 7g runs out of its exhaustive search on
    the empty single GPU of node 0 (rank 0) and fails on the full node 1 (rank 1) before it takes node 2 (rank 2); its
    later pairs on nodes 0 and 1 are dry runs, the one on node 2 OK.  A second pod then fits node 0."""
    R, api = pkg.records, pkg.api
    from test_pod_mode import _mig
    g, off = R.make_inventory([1, 1, 2], mig=True)
    g["busy"][1] = 0xFF
    w = SimpleNamespace(gpus=g, node_off=off, table=R.default_table(), n_node=3)
    c = np.concatenate([_mig(R, [R.GI_1_SLICE] * 7 + [R.GI_7_SLICE]), _mig(R, [R.GI_1_SLICE])])
    pod_off = np.array([0, 8, 9], np.uint32)
    W = _world(pkg, w, 3, [0, 1, 2, 3], 2)
    try:
        for cands in ([[0, 1, 2, 0, 1, 2], [2, 0]], [[1, 0, 2, 2, 1, 0], [0, 1, 2]]):
            cn, co = _flat(cands)
            for flags in (api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY, api.F_FRESH_INVENTORY):
                ref = _check(W, w, c, pod_off, cn, co, None, 9, flags, f"cands {cands} flags {flags}")
                if ref[1][0] == 2:
                    k = int(np.flatnonzero(cn[:co[1]] == 2)[0])
                    assert (ref[3][k + 1:co[1]][cn[k + 1:co[1]] == 2] == Y.ST_OK).all()
                if flags & api.F_EXHAUSTIVE:
                    assert Y.ST_SEARCH_LIMIT in ref[3][:co[1]].tolist()
    finally:
        W.close()


def test_windows_wider_than_the_resident_warps(pkg):
    """10,000 nodes over two ranks on one device: each warp cycles over several nodes and answers long runs of dry runs.
    Every output against dra_place_pods_why_batch on one context holding the same inventory."""
    api = pkg.api
    rng = np.random.default_rng(21)
    w, pod_off = pkg.synth.pods(10_000, 10_000, 21)
    n_pod = len(pod_off) - 1
    cn = rng.integers(0, w.n_node + 2, n_pod * 8).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 8).astype(np.uint32)
    W = _world(pkg, w, 2, [0, 5000, 10_000], 0, max_pods=n_pod, max_pairs=n_pod * 8)
    with api.Context(device=0) as single:
        single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
        try:
            for flags in (api.F_FRESH_INVENTORY, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY):
                res = _why(W, w.claims, pod_off, (cn, co), None, len(w.claims), flags)
                ref = single.place_pods_why(w.claims, pod_off, cn, co, None, len(w.claims), flags)
                for r, (table, got) in enumerate(res):
                    assert table.tobytes() == ref[0].tobytes(), f"flags {flags} rank {r}"
                    S.same(got, [ref[1]] + list(ref[2:]), NAMES, f"10k nodes flags {flags} rank {r}")
                assert (ref[2] == Y.ST_OK).any() and (ref[1] != NONE).any()
        finally:
            W.close()


def test_world1_equals_single_inventory_call(pkg):
    """World 1 over [0, n_node), no export: every output and the inventory byte for byte dra_place_pods_why_batch's."""
    api = pkg.api
    rng = np.random.default_rng(3)
    w, pod_off = pkg.synth.pods(400, 13, 13)
    n_pod = len(pod_off) - 1
    cn = rng.integers(0, w.n_node + 2, n_pod * 8).astype(np.uint32)
    co = (np.arange(n_pod + 1) * 8).astype(np.uint32)
    W = _world(pkg, w, 1, [0, w.n_node], 0)
    with api.Context(device=0) as single:
        single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
        try:
            for flags in _flags(api):
                for c_, o_ in ((cn, co), (None, None)):
                    (table, got), = _why(W, w.claims, pod_off, None if o_ is None else (c_, o_), None, len(w.claims), flags)
                    ref = single.place_pods_why(w.claims, pod_off, c_, o_, None, len(w.claims), flags)
                    assert table.tobytes() == ref[0].tobytes()
                    S.same(got, [ref[1]] + list(ref[2:]), NAMES, f"world 1 flags {flags}")
                    assert W.ctxs[0].get_inventory().tobytes() == single.get_inventory().tobytes(), f"flags {flags}"
            assert W.ctxs[0].last_chain() == {"place_shard", "place_why"}
        finally:
            W.close()


def test_calls_interleaved_on_one_world(pkg):
    """One world of three ranks, each call checked: the reasons call, sharded place pods, sharded reasons of UnsuitableNodes
    (the same exchange region, so the call parity must advance alike), the reasons call again, sharded pods Allocate,
    the inventory sync, the reasons call, and the sharded Deallocate of its table."""
    api = pkg.api
    rng = np.random.default_rng(41)
    w, pod_off = pkg.synth.pods(300, 12, 41)
    n_pod = len(pod_off) - 1
    bounds = S.bounds(w.n_node, 3, "uneven")
    W = _world(pkg, w, 3, bounds, 1)
    try:
        cn, co = S.candidates(rng, n_pod, w.n_node)
        _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), api.F_EXHAUSTIVE, "first")
        ref, ref_node, _ = P.place_pods(W.state(), w.node_off, w.table, w.claims, pod_off, None, None, None, len(w.claims), 0)
        for table, node in S.place(W, w.claims, pod_off, None, None, len(w.claims)):
            assert table.tobytes() == ref.tobytes() and node.tobytes() == ref_node.tobytes()
        for it in range(3):                              # §17's calls on the shared region, an odd and an even number
            state = W.state()
            sub = pod_off[: 40 + it + 1]
            yref = Y.why(state, w.node_off, w.table, w.claims[: int(sub[-1])], sub, cn, co[: len(sub)], 0)
            from test_gpu_shard_unsuitable_why import _why as uwhy
            for got in uwhy(W, w.claims[: int(sub[-1])], sub, (cn, co[: len(sub)])):
                S.same(got, yref, ("pair_why", "pair_claim", "pod_why", "claim_blocks"), f"§17 call {it}")
            _check(W, w, w.claims, pod_off, None, None, None, len(w.claims), 0, f"after {it + 1} §17 calls")
        run_off = np.arange(0, 61, 3, dtype=np.uint32)
        S.pods(W, w.claims[:60], run_off, None, 60)
        _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), api.F_EXHAUSTIVE, "after pods Allocate")
        W.sync_inventory()
        state = W.state()
        for inv in W.inventories():
            assert inv.tobytes() == state.tobytes()
        ref = _check(W, w, w.claims, pod_off, None, None, None, len(w.claims), 0, "after the sync")
        placed = w.claims.copy()
        for p in range(n_pod):
            placed["node"][pod_off[p]: pod_off[p + 1]] = ref[1][p] if ref[1][p] != NONE else 0
        S.deallocate(W, placed, None, len(placed), state=state, what="release", out=ref[0])
        assert W.state().tobytes() == state.tobytes()
        _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), 0, "after the release")
    finally:
        W.close()


@pytest.mark.parametrize("kind", ["pod_off order", "pod_off span", "cand_off order", "cand_off span", "packet room"])
def test_device_faults_fail_every_rank(pkg, kind):
    """A fault found on the device fails the call on every rank with none of the reason outputs written (claim_blocks
    included) and no inventory word changed; the next call on the same world is right."""
    api = pkg.api
    w, pod_off = pkg.synth.pods(120, 11, 3)
    n_pod = len(pod_off) - 1
    cn, co = S.cands(np.random.default_rng(0), n_pod, w.n_node, 4)
    W = _world(pkg, w, 3, S.bounds(w.n_node, 3, "uneven"), 1, cap_per_rank=8 if kind == "packet room" else 0)
    try:
        po, co_ = pod_off.copy(), co.copy()
        if kind == "pod_off order":
            po[5] = po[6] + 1
        elif kind == "pod_off span":
            po[-1] -= 1
        elif kind == "cand_off order":
            co_[3] = co_[4] + 2
        elif kind == "cand_off span":
            co_[0] = 1
        for flags in (0, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY):
            for cands in ((cn, co_),) if kind.startswith("cand") else ((cn, co_), None):
                before = W.inventories()
                outs = _why(W, w.claims, po, cands, None, len(w.claims), flags, expect=api.E_INVAL)
                for r, o in enumerate(outs):
                    for name, h in zip(NAMES[1:], o[1:]):
                        assert (h == SENTINEL).all(), f"{kind} flags {flags}: rank {r} wrote {name}"
                for b, a in zip(before, W.inventories()):
                    assert a.tobytes() == b.tobytes(), f"{kind}: a failed call changed an inventory"
        if kind != "packet room":
            _check(W, w, w.claims, pod_off, cn, co, None, len(w.claims), api.F_EXHAUSTIVE, f"after {kind}")
        else:
            one = np.array([0, int(pod_off[1])], np.uint32)
            _check(W, w, w.claims[: one[1]], one, cn[:4], co[:2], None, int(one[1]), 0, "within the packet room")
    finally:
        W.close()


def test_host_refusals(pkg):
    """Host-side refusals return before anything is enqueued; a valid call enqueues the sharded place pods' kernels plus
    the reasons' prep, push and merge."""
    import torch
    api = pkg.api
    w, pod_off = pkg.synth.pods(60, 11, 3)
    n_pod = len(pod_off) - 1
    bounds = [0, 5, 11]
    cn, co = S.cands(np.random.default_rng(1), n_pod, w.n_node, 4)
    d_c, d_p, d_n, d_o, d_pn = S.dev(w.claims), S.dev(pod_off), S.dev(cn), S.dev(co), S.dev(np.zeros(n_pod, np.uint32))
    sentinel = torch.full((1 << 14,), SENTINEL, dtype=torch.uint8, device="cuda:0")
    o = sentinel.data_ptr()
    torch.cuda.synchronize()

    def raw(c, **k):
        a = dict(claims=d_c.data_ptr(), n_claim=len(w.claims), pod_off=d_p.data_ptr(), n_pod=n_pod, cn=d_n.data_ptr(),
                 co=d_o.data_ptr(), n_pair=len(cn), out_off=None, n_out=len(w.claims), pod_node=d_pn.data_ptr(), why=o,
                 flags=0)
        a.update(k)
        return c._lib.dra_place_pods_why_batch_global_device(c._h, a["claims"], a["n_claim"], a["pod_off"], a["n_pod"], a["cn"],
                                                             a["co"], a["n_pair"], a["out_off"], a["n_out"], a["pod_node"],
                                                             a["why"], o, o, o, a["flags"])

    W = _world(pkg, w, 2, bounds, 1, max_pods=n_pod, max_pairs=len(cn))
    try:
        c0 = W.ctxs[0]
        launches = c0.launch_count()
        assert raw(c0, flags=0x80) == api.E_INVAL                            # unknown flag
        assert raw(c0, n_out=N_OUT_MAX + 1) == api.E_INVAL                   # past the exported table
        assert raw(c0, cn=None) == api.E_INVAL                               # candidates: both or neither
        assert raw(c0, cn=None, co=None) == api.E_INVAL                      # dense form with n_pair != 0
        assert raw(c0, cn=None, co=None, n_pair=0) == api.E_INVAL            # dense: n_pod * n_node above max_pairs
        assert raw(c0, n_pair=len(cn) + 1) == api.E_INVAL                    # above max_pairs
        assert raw(c0, n_pod=n_pod + 1) == api.E_STATE                       # beyond max_pods of the export
        assert raw(c0, why=None) == api.E_INVAL                              # pairs to answer and no pair_why
        assert raw(c0, pod_node=None) == api.E_INVAL
        assert c0.launch_count() == launches
        torch.cuda.synchronize()
        assert (sentinel.cpu().numpy() == SENTINEL).all(), "a refused call wrote an output"
        # a valid call's launches: the sharded place pods' plus the reasons' prep, push and merge
        l0 = [c.launch_count() for c in W.ctxs]
        S.place(W, w.claims, pod_off, (cn, co), None, len(w.claims))
        l1 = [c.launch_count() for c in W.ctxs]
        _why(W, w.claims, pod_off, (cn, co), None, len(w.claims))
        l2 = [c.launch_count() for c in W.ctxs]
        assert [b - a - (c - b) for a, b, c in zip(l0, l1, l2)] == [-3] * 2
        assert {"place_shard", "place_why"} <= c0.last_chain()
    finally:
        W.close()
    # a world exported without the reasons' room: DRA_E_STATE, even with no pairs, nothing enqueued
    W = _world(pkg, w, 2, bounds, 1, max_pods=n_pod, max_pairs=None)
    try:
        c0 = W.ctxs[0]
        launches = c0.launch_count()
        assert raw(c0) == api.E_STATE
        assert raw(c0, co=S.dev(np.zeros(n_pod + 1, np.uint32)).data_ptr(), n_pair=0) == api.E_STATE
        assert c0.launch_count() == launches
    finally:
        W.close()
    # dense n_pod * n_node >= 2^32 on one inventory of 70 nodes (2^26 pods, the most the sharded call takes)
    w70, _ = pkg.synth.pods(100, 70, 3)
    W = _world(pkg, w70, 1, [0, w70.n_node], 0)
    try:
        c0 = W.ctxs[0]
        launches = c0.launch_count()
        assert raw(c0, cn=None, co=None, n_pair=0, n_pod=1 << 26, n_claim=0, n_out=0) == api.E_INVAL
        assert c0.launch_count() == launches
    finally:
        W.close()


def test_multi_process():
    """tests/multi_gpu_shard_place_why_check.py under torchrun, one process per GPU with IPC-mapped peer buffers."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    from test_gpu_multi_rank import _free_port
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={min(n, 4)}",
                        "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                        os.path.join(ROOT, "tests", "multi_gpu_shard_place_why_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
