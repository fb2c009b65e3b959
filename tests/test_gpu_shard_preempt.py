"""GPU suite: preemption on a sharded world (dra_preempt_batch_global_device, spec §14 "Sharded form").  World contexts of
this process on ONE device, wired with dra_comm_init_local / dra_peer_import_local like test_gpu_shard_unsuitable.py.
Every rank's six outputs must be byte for byte the oracle's answer on the world's state: the inventory each rank holds for
its own node range."""
import numpy as np
import pytest

import preempt_oracle as P
import shard_world as S
from shard_world import Running

pytestmark = pytest.mark.gpu
SENTINEL = 0x5C
NAMES = S.PREEMPT_NAMES[:6]
SIZES = (4096, 200000, 64)                               # max_pods, max_pairs, max_victims


def _world(pkg, w, world, bounds, invs=None, sizes=SIZES, n_out=None, **kw):
    """rank r serving [bounds[r], bounds[r+1]) of the inventory it was given, preemption and its pairs reserved"""
    return S.World(pkg, w.table, w.node_off, w.gpus if invs is None else invs, world, bounds,
                   n_out_max=max(1, n_out or len(w.run_claims)), preempt=sizes, pairs=sizes[1], **kw)


def _oracle(pkg, gpus, w, claims, pod_off, prio, cands, max_victims, flags, run=None):
    rc, rpo, rpr, ro = run if run is not None else (w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    cn, co = (None, None) if cands is None else cands
    return P.preempt(gpus, w.node_off, w.table, claims, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, max_victims,
                     P.F_EXHAUSTIVE if flags & pkg.api.F_EXHAUSTIVE else 0)


def _running(pkg, w):
    return Running(pkg, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)


def _check_all(pkg, W, w, run, combos, rng, what):
    for flags, form, mv, pairs in combos:
        n_pod = len(w.pod_off) - 1
        cands = None if form == "dense" else S.cands(rng, n_pod, S.nn(w), 16)
        ref = _oracle(pkg, W.state(), w, w.claims, w.pod_off, w.prio, cands, mv, flags)
        for r, got in enumerate(S.preempt(W, w.claims, w.pod_off, w.prio, run, cands, mv, flags, pairs)):
            S.same(got, ref, NAMES, f"{what} rank {r} f{flags} {form} mv{mv} pairs{pairs}")


COMBOS = [(0, "dense", 16, True), (1, "cands", 3, False), (0, "cands", 0, True), (1, "dense", 3, False),
          (1, "cands", 16, True), (0, "dense", 0, False)]


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven"),
                                        (4, "even"), (4, "empty")])
@pytest.mark.parametrize("width", [4, 8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    """Every form, flag, row width and pair-output choice, every rank's outputs against the oracle."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=60, seed=world * 10 + width)
    combos = [(f * pkg.api.F_EXHAUSTIVE, form, mv, pairs) for f, form, mv, pairs in COMBOS]
    W = _world(pkg, w, world, S.bounds(S.nn(w), world, kind))
    try:
        run = _running(pkg, w)
        _check_all(pkg, W, w, run, combos, np.random.default_rng(world + width), f"w{world} {kind} width {width}")
        got = S.preempt(W, w.claims, w.pod_off, w.prio, run)[0]
        assert (got[3] == P.EVICT).any() and (got[0] == P.EVICT).any()
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_shared_heavy_world(pkg, world):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=60, seed=4, mig_nodes=0)
    W = _world(pkg, w, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        combos = [(f, form, 16, True) for f in (0, pkg.api.F_EXHAUSTIVE) for form in ("dense", "cands")]
        _check_all(pkg, W, w, _running(pkg, w), combos, np.random.default_rng(3), f"shared w{world}")
    finally:
        W.close()


def test_selectors_and_long_pods(pkg):
    R = pkg.records
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=30, seed=7)
    attrs = np.zeros(len(w.gpus), R.ATTR_DTYPE)
    attrs["index"] = np.arange(len(w.gpus)) % 8
    attrs["mem_total_mib"] = 81920
    sels = np.stack([R.selector(("cmp", R.ATTR_INDEX, R.CMP_LT, 4)), R.selector(("cmp", R.ATTR_INDEX, R.CMP_GE, 4))])
    c = w.claims.copy()
    mig = c["kind"] == R.KIND_MIG
    c["mem_limit_mib"] = np.where(mig, (np.arange(len(c)) % 4).astype(np.uint32), 0)   # ids 0..3, 3 beyond the table
    extra = np.zeros(65, R.CLAIM_DTYPE)                   # a pod of 32 1g claims and one of 33
    extra["kind"], extra["count"], extra["profile"] = R.KIND_MIG, 1, R.GI_1_SLICE
    c = np.concatenate([c, extra])
    pod_off = np.concatenate([w.pod_off, [len(w.claims) + 32, len(c)]]).astype(np.uint32)
    prio = np.concatenate([w.prio, [2000, 2000]]).astype(np.int32)
    W = _world(pkg, w, 3, S.bounds(S.nn(w), 3, "uneven"), attrs=attrs, sels=sels)
    P.set_selectors(attrs, sels)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(1)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for cands in (None, S.cands(rng, len(pod_off) - 1, S.nn(w), 5)):
                ref = _oracle(pkg, W.state(), w, c, pod_off, prio, cands, 16, flags)
                for r, got in enumerate(S.preempt(W, c, pod_off, prio, run, cands, 16, flags)):
                    S.same(got, ref, NAMES, f"selectors rank {r} f{flags}")
                    assert got[3][-1] == P.INVALID
    finally:
        P.set_selectors()
        W.close()


def test_diverged_copies(pkg):
    """Each rank holds the real world on its own range only, the empty inventory elsewhere: the sharded answer is the
    oracle's on the real world, while rank 0's dra_preempt_batch (its own copy taken for the world) is not."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=60, seed=21)
    world = 3
    bounds = S.bounds(S.nn(w), world, "even")
    invs = []
    for r in range(world):
        g = w.empty.copy()
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        g[a:b] = w.gpus[a:b]
        invs.append(g)
    W = _world(pkg, w, world, bounds, invs=invs)
    try:
        assert W.state().tobytes() == w.gpus.tobytes()
        run = _running(pkg, w)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            ref = _oracle(pkg, w.gpus, w, w.claims, w.pod_off, w.prio, None, 16, flags)
            for r, got in enumerate(S.preempt(W, w.claims, w.pod_off, w.prio, run, None, 16, flags)):
                S.same(got, ref, NAMES, f"diverged rank {r} f{flags}")
            single = W.ctxs[0].preempt(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                                       max_victims=16, flags=flags)
            assert any(x.tobytes() != y.tobytes() for x, y in zip(single, ref)), "the workload does not expose stale copies"
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == invs[r].tobytes(), f"rank {r}'s inventory changed"
    finally:
        W.close()


def test_the_real_flow(pkg):
    """The running pods are placed by the sharded pods Allocate, with no sync before the preemption call, and their
    records are the gathered table; no inventory word, live or pristine, changes in the preemption call."""
    R = pkg.records
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=50, seed=13)
    world = 3
    bounds = S.bounds(S.nn(w), world, "uneven")
    n_out = len(w.run_claims)
    W = _world(pkg, w, world, bounds, invs=[w.empty] * world, n_out=n_out)
    try:
        import torch
        rc = w.run_claims.copy()
        d_rc, d_rpo = S.dev(rc), S.dev(w.run_pod_off)
        torch.cuda.synchronize()
        for c in W.ctxs:
            c.allocate_pods_global_device(d_rc.data_ptr(), len(rc), d_rpo.data_ptr(), len(w.run_pod_off) - 1, None, n_out, 0)
        runs = [Running(pkg, rc, w.run_pod_off, w.run_prio, w.run_out, out_ptr=S.table_ptr(c)) for c in W.ctxs]
        got_all = S.preempt(W, w.claims, w.pod_off, w.prio, runs, None, 16, 0)
        table = W.ctxs[0].gather_read(np.zeros(n_out, R.OUT_DTYPE))
        assert (table["status"] == R.ST_OK).sum() > n_out // 2
        state = W.state()
        befores = [c.get_inventory() for c in W.ctxs]
        ref = _oracle(pkg, state, w, w.claims, w.pod_off, w.prio, None, 16, 0, run=(rc, w.run_pod_off, w.run_prio, table))
        for r, got in enumerate(got_all):
            S.same(got, ref, NAMES, f"real flow rank {r}")
        assert (ref[3] == P.EVICT).any()
        # another call on the same state: the inventories stay as the pods Allocate left them; the pristine copies too
        for r, got in enumerate(S.preempt(W, w.claims, w.pod_off, w.prio, runs[0], None, 16, pkg.api.F_EXHAUSTIVE)):
            S.same(got, _oracle(pkg, state, w, w.claims, w.pod_off, w.prio, None, 16, pkg.api.F_EXHAUSTIVE,
                               run=(rc, w.run_pod_off, w.run_prio, table)), NAMES, f"real flow again rank {r}")
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == befores[r].tobytes(), f"rank {r}: live inventory changed"
            c.reset_inventory()
            assert c.get_inventory().tobytes() == w.empty.tobytes(), f"rank {r}: pristine inventory changed"
    finally:
        W.close()


def test_world_one_is_the_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=80, seed=2)
    W = _world(pkg, w, 1, [0, S.nn(w)], export=False)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(0)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for cands in (None, S.cands(rng, len(w.pod_off) - 1, S.nn(w), 7)):
                cn, co = (None, None) if cands is None else cands
                single = W.ctxs[0].preempt(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio,
                                           w.run_out, None, cn, co, 8, flags)
                S.same(S.preempt(W, w.claims, w.pod_off, w.prio, run, cands, 8, flags)[0], single, NAMES, f"world 1 f{flags}")
        assert "preempt_shard" in W.ctxs[0].last_chain()
    finally:
        W.close()


def test_consecutive_calls_of_changing_size(pkg):
    """Calls of growing and shrinking size, interleaved with sharded UnsuitableNodes, pods Allocate and the inventory
    sync on the same world: call parity and the shared peer buffer."""
    import torch
    R = pkg.records
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=120, seed=31, fill=60)
    world = 4
    bounds = S.bounds(S.nn(w), world, "uneven")
    W = _world(pkg, w, world, bounds, n_out=4096)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(8)
        for it, n in enumerate((40, 120, 7, 90, 1, 120)):
            po = w.pod_off[: n + 1]
            claims = w.claims[: int(po[-1])]
            prio = w.prio[:n]
            flags = pkg.api.F_EXHAUSTIVE if it % 2 else 0
            cands = None if it % 3 == 0 else S.cands(rng, n, S.nn(w), 1 + it)
            mv = (0, 3, 16)[it % 3]
            ref = _oracle(pkg, W.state(), w, claims, po, prio, cands, mv, flags)
            for r, got in enumerate(S.preempt(W, claims, po, prio, run, cands, mv, flags, pairs=it % 2 == 0)):
                S.same(got, ref, NAMES, f"call {it} rank {r}")
            # sharded UnsuitableNodes on the same buffer
            bits = S.unsuitable(W, claims, po, flags=flags)
            assert all(b.tobytes() == bits[0].tobytes() for b in bits)
            # pods Allocate of a few pending pods onto their first candidate's node, then the inventory sync
            pod = w.claims[w.pod_off[it]: w.pod_off[it + 1]].copy()
            pod["node"] = (it * 5) % S.nn(w)
            oo, n_out = R.out_offsets(pod, S.nn(w))
            d_pod, d_ppo, d_oo = S.dev(pod), S.dev(np.array([0, len(pod)], np.uint32)), S.dev(oo)
            torch.cuda.synchronize()
            for c in W.ctxs:                              # the pods Allocate and the sync enqueued with no wait between
                c.allocate_pods_global_device(d_pod.data_ptr(), len(pod), d_ppo.data_ptr(), 1, d_oo.data_ptr(), n_out, 0)
            W.sync_inventory()
    finally:
        W.close()


def _bad_running(w, kind):
    ST_OK = 0                                             # records.ST_OK
    rc, rpo, rpr, ro = w.run_claims.copy(), w.run_pod_off.copy(), w.run_prio.copy(), w.run_out.copy()
    if kind == "running pod_off":
        rpo[2] = rpo[3] + 1
    elif kind == "slot outside n_out":
        ro = ro[:-1]
    elif kind == "gpu >= n_gpu":
        ok = np.flatnonzero(ro["status"] == ST_OK)
        ro["gpu"][ok[0]] = len(w.gpus) + 3
    elif kind == "two nodes":
        multi = [p for p in range(len(rpo) - 1) if rpo[p + 1] - rpo[p] >= 2]
        if multi:
            i = int(rpo[multi[0]])
            ro["gpu"][i + 1] = (int(ro["gpu"][i]) + 8 * 3) % len(w.gpus)
            ro["status"][i: i + 2] = ST_OK
        else:                                             # one pod takes over the next pod's slot range as well
            rc = np.concatenate([rc[:1], rc])
            ro = np.concatenate([ro[:1], ro])
            ro["gpu"][1] = (int(ro["gpu"][0]) + 8 * 3) % len(w.gpus)
            ro["status"][:2] = ST_OK
            rpo = np.concatenate([[0], rpo[1:] + 1]).astype(np.uint32)
    return rc, rpo, rpr, ro


@pytest.mark.parametrize("kind", ["pod_off", "cand_off", "running pod_off", "slot outside n_out", "gpu >= n_gpu",
                                  "two nodes"])
def test_device_faults_fail_every_rank(pkg, kind):
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=17)
    world = 3
    W = _world(pkg, w, world, S.bounds(S.nn(w), world, "uneven"))
    try:
        po, cands = w.pod_off.copy(), None
        rc, rpo, rpr, ro = w.run_claims, w.run_pod_off, w.run_prio, w.run_out
        if kind == "pod_off":
            po[5] = po[6] + 1
        elif kind == "cand_off":
            cn, co = S.cands(np.random.default_rng(0), len(po) - 1, S.nn(w), 4)
            co[3] = co[4] + 2
            cands = (cn, co)
        else:
            rc, rpo, rpr, ro = _bad_running(w, kind)
        run = Running(pkg, rc, rpo, rpr, ro)
        outs = S.preempt(W, w.claims, po, w.prio, run, cands, 16, 0, expect=A.E_INVAL)
        for r, o in enumerate(outs):
            assert all((h == SENTINEL).all() for h in o), f"{kind}: rank {r} wrote an output"
        # the next valid call on the same world matches the oracle
        _check_all(pkg, W, w, _running(pkg, w), [(0, "cands", 16, True)], np.random.default_rng(2), f"after {kind}")
    finally:
        W.close()


def test_host_side_errors(pkg):
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=5)
    n_pod = len(w.pod_off) - 1
    W = _world(pkg, w, 2, S.bounds(S.nn(w), 2, "even"), sizes=(n_pod, n_pod * S.nn(w), 8))
    try:
        run = _running(pkg, w)
        c = W.ctxs[0]
        import torch
        keep = [S.dev(w.claims), S.dev(w.pod_off), S.dev(w.prio)]
        o = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda:0").data_ptr()
        n_pair = n_pod * S.nn(w)
        launches = c._lib.dra_launch_count(c._h)

        def call(n_pair=n_pair, mv=8, victims=o, flags=0, ctx=c, n=n_pod):
            with pytest.raises(A.DraError) as e:
                ctx.preempt_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n,
                                          None, None, n_pair, run.struct, o, o, o, o, o, victims, mv, flags)
            return e.value.code

        assert call(flags=0x2) == A.E_INVAL                                   # unknown flags
        assert call(victims=None) == A.E_INVAL                                # max_victims without a buffer
        assert call(mv=9) == A.E_INVAL                                        # above the export's max_victims
        assert call(n_pair=n_pair + 1) == A.E_INVAL                           # dense n_pair != n_pod * n_node
        assert c._lib.dra_launch_count(c._h) == launches
    finally:
        W.close()
    # sizes above the export's: more pods than max_pods
    W = _world(pkg, w, 2, S.bounds(S.nn(w), 2, "even"), sizes=(n_pod - 1, n_pod * S.nn(w), 8))
    try:
        with pytest.raises(A.DraError) as e:
            S.preempt(W, w.claims, w.pod_off, w.prio, _running(pkg, w), None, 8)
        assert e.value.code == A.E_INVAL
    finally:
        W.close()
    # a bare dra_set_shard, and a world with no export
    for kw in (dict(bare=True), dict(export=False)):
        W = _world(pkg, w, 2, S.bounds(S.nn(w), 2, "even"), **kw)
        try:
            with pytest.raises(A.DraError) as e:
                S.preempt(W, w.claims, w.pod_off, w.prio, _running(pkg, w), None, 8)
            assert e.value.code == A.E_STATE, kw
        finally:
            W.close()
