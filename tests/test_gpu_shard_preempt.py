"""GPU suite: preemption on a sharded world (dra_preempt_batch_global_device, spec §14 "Sharded form").  World contexts of
this process on ONE device, wired with dra_comm_init_local / dra_peer_import_local like test_gpu_shard_unsuitable.py.
Every rank's six outputs must be byte for byte the oracle's answer on the world's state: the inventory each rank holds for
its own node range."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_shard_unsuitable import _bounds

import preempt_oracle as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFF
SENTINEL = 0x5C
NAMES = ("pair_status", "pair_victims", "pod_node", "pod_status", "n_victims", "victims")


def _dev(a):
    import torch
    a = np.ascontiguousarray(a)
    if a.nbytes == 0:
        return torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to("cuda:0")


def _nn(w):
    return len(w.node_off) - 1


class Running:
    """The running pods on the device, and the dra_running_pods struct pointing at them."""

    def __init__(self, pkg, claims, pod_off, prio, out, out_off=None, out_ptr=None):
        self.keep = [_dev(claims), _dev(pod_off), _dev(prio), _dev(out)] + ([_dev(out_off)] if out_off is not None else [])
        self.struct = pkg.api.RunningPods(self.keep[0].data_ptr(), len(claims), self.keep[1].data_ptr(), len(pod_off) - 1,
                                          self.keep[2].data_ptr(), self.keep[4].data_ptr() if out_off is not None else None,
                                          out_ptr if out_ptr is not None else self.keep[3].data_ptr(), len(out))


class World:
    """world contexts on device 0, rank r serving [bounds[r], bounds[r+1]) of the inventory it was given."""

    def __init__(self, pkg, w, world, bounds, invs=None, sizes=(4096, 200000, 64), attrs=None, sels=None, export=True,
                 bare=False, n_out=None):
        R = pkg.records
        self.pkg, self.w, self.world, self.bounds = pkg, w, world, list(bounds)
        self.ctxs = [pkg.api.Context(device=0) for _ in range(world)]
        for r, c in enumerate(self.ctxs):
            c.comm_init_local(r, world)
            c.set_table(w.table)
            c.set_inventory(w.gpus if invs is None else invs[r], w.node_off)
            if sels is not None:
                c.set_gpu_attrs(attrs); c.set_selectors(sels.reshape(-1, R.SEL_MAX_INS))
            if bare:
                c.set_shard(bounds[r], bounds[r + 1], r == 0)
            else:
                c.set_shard_map(bounds, stray_rank=0)
            if world > 1 and export:
                c.set_shard_preempt(*sizes)
                c.set_shard_pairs(sizes[1])
                c.shard_export(max(1, n_out or len(w.run_claims)), 0, want_handle=False)
        if world > 1 and export:
            for c in self.ctxs:
                c.peer_import_local(self.ctxs)

    def close(self):
        for c in self.ctxs:
            c.close()

    def state(self):
        """the world's state: each rank's own GPU range as that rank holds it"""
        g = self.w.gpus.copy()
        for r, c in enumerate(self.ctxs):
            a, b = int(self.w.node_off[self.bounds[r]]), int(self.w.node_off[self.bounds[r + 1]])
            g[a:b] = c.get_inventory()[a:b]
        return g

    def enqueue(self, claims, pod_off, prio, run, cands=None, max_victims=16, flags=0, pairs=True, victims_buf=True):
        """The call on every rank (enqueued on all of them first); returns (per-rank sentinel-filled outputs, keep)."""
        import torch
        n_pod = len(pod_off) - 1
        cn, co = (None, None) if cands is None else cands
        n_pair = n_pod * _nn(self.w) if co is None else int(co[-1])
        keep = [_dev(claims), _dev(pod_off), _dev(prio)]
        keep += [None, None] if cn is None else [_dev(cn), _dev(co)]
        sizes = (n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * max_victims * 4)
        outs = [[torch.full((s + 16,), SENTINEL, dtype=torch.uint8, device="cuda:0") for s in sizes] for _ in self.ctxs]
        torch.cuda.synchronize()                         # (the contexts' streams do not wait for torch's)
        ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        for c, o in zip(self.ctxs, outs):
            c.preempt_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                    ptr(keep[3]), ptr(keep[4]), n_pair, run.struct,
                                    o[0].data_ptr() if pairs else None, o[1].data_ptr() if pairs else None,
                                    o[2].data_ptr(), o[3].data_ptr(), o[4].data_ptr(),
                                    o[5].data_ptr() if victims_buf and max_victims else None, max_victims, flags)
        return outs, (keep, sizes, n_pod)

    def read(self, outs, meta, pairs=True, max_victims=16):
        """each rank's outputs as the oracle returns them, checking that nothing was written past them"""
        keep, sizes, n_pod = meta
        res = []
        for r, o in enumerate(outs):
            hs = [t.cpu().numpy() for t in o]
            for i, (h, s) in enumerate(zip(hs, sizes)):
                assert (h[s:] == SENTINEL).all(), f"rank {r} wrote past {NAMES[i]}"
                if not pairs and i < 2:
                    assert (h == SENTINEL).all(), f"rank {r} wrote {NAMES[i]} without being asked"
            dt = (np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32)
            got = [h[:s].view(d) for h, s, d in zip(hs, sizes, dt)]
            got[5] = got[5].reshape(n_pod, max_victims)
            res.append(got)
        return res

    def call(self, claims, pod_off, prio, run, cands=None, max_victims=16, flags=0, pairs=True):
        outs, meta = self.enqueue(claims, pod_off, prio, run, cands, max_victims, flags, pairs)
        for c in self.ctxs:
            c.sync()
        return self.read(outs, meta, pairs, max_victims)


def _oracle(pkg, gpus, w, claims, pod_off, prio, cands, max_victims, flags, run=None):
    rc, rpo, rpr, ro = run if run is not None else (w.run_claims, w.run_pod_off, w.run_prio, w.run_out)
    cn, co = (None, None) if cands is None else cands
    return P.preempt(gpus, w.node_off, w.table, claims, pod_off, prio, rc, rpo, rpr, ro, None, cn, co, max_victims,
                     P.F_EXHAUSTIVE if flags & pkg.api.F_EXHAUSTIVE else 0)


def _same(got, ref, what, pairs=True):
    for i, (name, x, y) in enumerate(zip(NAMES, got, ref)):
        if not pairs and i < 2:
            continue
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.reshape(-1) != y.reshape(-1))[:5]
            pytest.fail(f"{what}: {name} differs at {bad}: device {x.reshape(-1)[bad]} oracle {y.reshape(-1)[bad]}")


def _cands(rng, n_pod, n_node, k):
    nodes = rng.integers(0, n_node + 3, size=n_pod * k).astype(np.uint32)       # duplicates and strays included
    if len(nodes) > 3:
        nodes[1] = nodes[0]
        nodes[2] = NONE
    return nodes, (np.arange(n_pod + 1) * k).astype(np.uint32)


def _running(pkg, w):
    return Running(pkg, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)


def _check_all(pkg, W, w, run, combos, rng, what):
    for flags, form, mv, pairs in combos:
        n_pod = len(w.pod_off) - 1
        cands = None if form == "dense" else _cands(rng, n_pod, _nn(w), 16)
        ref = _oracle(pkg, W.state(), w, w.claims, w.pod_off, w.prio, cands, mv, flags)
        for r, got in enumerate(W.call(w.claims, w.pod_off, w.prio, run, cands, mv, flags, pairs)):
            _same(got, ref, f"{what} rank {r} f{flags} {form} mv{mv} pairs{pairs}", pairs)


COMBOS = [(0, "dense", 16, True), (1, "cands", 3, False), (0, "cands", 0, True), (1, "dense", 3, False),
          (1, "cands", 16, True), (0, "dense", 0, False)]


@pytest.mark.parametrize("world,kind", [(1, "even"), (2, "even"), (2, "uneven"), (3, "empty"), (3, "uneven"),
                                        (4, "even"), (4, "empty")])
@pytest.mark.parametrize("width", [4, 8, 16, 32])
def test_matches_oracle(pkg, world, kind, width):
    """Every form, flag, row width and pair-output choice, every rank's outputs against the oracle."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=width, n_pending=60, seed=world * 10 + width)
    combos = [(f * pkg.api.F_EXHAUSTIVE, form, mv, pairs) for f, form, mv, pairs in COMBOS]
    W = World(pkg, w, world, _bounds(_nn(w), world, kind))
    try:
        run = _running(pkg, w)
        _check_all(pkg, W, w, run, combos, np.random.default_rng(world + width), f"w{world} {kind} width {width}")
        got = W.call(w.claims, w.pod_off, w.prio, run)[0]
        assert (got[3] == P.EVICT).any() and (got[0] == P.EVICT).any()
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_shared_heavy_world(pkg, world):
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=60, seed=4, mig_nodes=0)
    W = World(pkg, w, world, _bounds(_nn(w), world, "uneven"))
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
    W = World(pkg, w, 3, _bounds(_nn(w), 3, "uneven"), attrs=attrs, sels=sels)
    P.set_selectors(attrs, sels)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(1)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for cands in (None, _cands(rng, len(pod_off) - 1, _nn(w), 5)):
                ref = _oracle(pkg, W.state(), w, c, pod_off, prio, cands, 16, flags)
                for r, got in enumerate(W.call(c, pod_off, prio, run, cands, 16, flags)):
                    _same(got, ref, f"selectors rank {r} f{flags}")
                    assert got[3][-1] == P.INVALID
    finally:
        P.set_selectors()
        W.close()


def test_diverged_copies(pkg):
    """Each rank holds the real world on its own range only, the empty inventory elsewhere: the sharded answer is the
    oracle's on the real world, while rank 0's dra_preempt_batch (its own copy taken for the world) is not."""
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=60, seed=21)
    world = 3
    bounds = _bounds(_nn(w), world, "even")
    invs = []
    for r in range(world):
        g = w.empty.copy()
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        g[a:b] = w.gpus[a:b]
        invs.append(g)
    W = World(pkg, w, world, bounds, invs=invs)
    try:
        assert W.state().tobytes() == w.gpus.tobytes()
        run = _running(pkg, w)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            ref = _oracle(pkg, w.gpus, w, w.claims, w.pod_off, w.prio, None, 16, flags)
            for r, got in enumerate(W.call(w.claims, w.pod_off, w.prio, run, None, 16, flags)):
                _same(got, ref, f"diverged rank {r} f{flags}")
            single = W.ctxs[0].preempt(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out,
                                       max_victims=16, flags=flags)
            assert any(x.tobytes() != y.tobytes() for x, y in zip(single, ref)), "the workload does not expose stale copies"
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == invs[r].tobytes(), f"rank {r}'s inventory changed"
    finally:
        W.close()


def _gather_ptr(ctx):
    p, n = C.c_void_p(), C.c_uint32()
    assert ctx._lib.dra_gather_table(ctx._h, C.byref(p), C.byref(n)) == 0
    return p.value


def test_the_real_flow(pkg):
    """The running pods are placed by the sharded pods Allocate, with no sync before the preemption call, and their
    records are the gathered table; no inventory word, live or pristine, changes in the preemption call."""
    R = pkg.records
    w = pkg.synth.preempt(n_node=24, gpus_per_node=8, n_pending=50, seed=13)
    world = 3
    bounds = _bounds(_nn(w), world, "uneven")
    n_out = len(w.run_claims)
    W = World(pkg, w, world, bounds, invs=[w.empty] * world, n_out=n_out)
    try:
        import torch
        rc = w.run_claims.copy()
        d_rc, d_rpo = _dev(rc), _dev(w.run_pod_off)
        torch.cuda.synchronize()
        for c in W.ctxs:
            c.allocate_pods_global_device(d_rc.data_ptr(), len(rc), d_rpo.data_ptr(), len(w.run_pod_off) - 1, None, n_out, 0)
        runs = [Running(pkg, rc, w.run_pod_off, w.run_prio, w.run_out, out_ptr=_gather_ptr(c)) for c in W.ctxs]
        keep = [_dev(w.claims), _dev(w.pod_off), _dev(w.prio)]
        n_pod = len(w.pod_off) - 1
        n_pair = n_pod * _nn(w)
        sizes = (n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * 16 * 4)
        outs = [[torch.full((s + 16,), SENTINEL, dtype=torch.uint8, device="cuda:0") for s in sizes] for _ in W.ctxs]
        torch.cuda.synchronize()
        for c, o, run in zip(W.ctxs, outs, runs):
            c.preempt_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                    None, None, n_pair, run.struct, *[t.data_ptr() for t in o], 16, 0)
        for c in W.ctxs:
            c.sync()
        got_all = W.read(outs, (keep, sizes, n_pod))
        table = W.ctxs[0].gather_read(np.zeros(n_out, R.OUT_DTYPE))
        assert (table["status"] == R.ST_OK).sum() > n_out // 2
        state = W.state()
        befores = [c.get_inventory() for c in W.ctxs]
        ref = _oracle(pkg, state, w, w.claims, w.pod_off, w.prio, None, 16, 0, run=(rc, w.run_pod_off, w.run_prio, table))
        for r, got in enumerate(got_all):
            _same(got, ref, f"real flow rank {r}")
        assert (ref[3] == P.EVICT).any()
        # another call on the same state: the inventories stay as the pods Allocate left them; the pristine copies too
        for r, got in enumerate(W.call(w.claims, w.pod_off, w.prio, runs[0], None, 16, pkg.api.F_EXHAUSTIVE)):
            _same(got, _oracle(pkg, state, w, w.claims, w.pod_off, w.prio, None, 16, pkg.api.F_EXHAUSTIVE,
                               run=(rc, w.run_pod_off, w.run_prio, table)), f"real flow again rank {r}")
        for r, c in enumerate(W.ctxs):
            assert c.get_inventory().tobytes() == befores[r].tobytes(), f"rank {r}: live inventory changed"
            c.reset_inventory()
            assert c.get_inventory().tobytes() == w.empty.tobytes(), f"rank {r}: pristine inventory changed"
    finally:
        W.close()


def test_world_one_is_the_single_inventory_call(pkg):
    w = pkg.synth.preempt(n_node=20, gpus_per_node=8, n_pending=80, seed=2)
    W = World(pkg, w, 1, [0, _nn(w)], export=False)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(0)
        for flags in (0, pkg.api.F_EXHAUSTIVE):
            for cands in (None, _cands(rng, len(w.pod_off) - 1, _nn(w), 7)):
                cn, co = (None, None) if cands is None else cands
                single = W.ctxs[0].preempt(w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio,
                                           w.run_out, None, cn, co, 8, flags)
                _same(W.call(w.claims, w.pod_off, w.prio, run, cands, 8, flags)[0], single, f"world 1 f{flags}")
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
    bounds = _bounds(_nn(w), world, "uneven")
    W = World(pkg, w, world, bounds, n_out=4096)
    try:
        run = _running(pkg, w)
        rng = np.random.default_rng(8)
        for it, n in enumerate((40, 120, 7, 90, 1, 120)):
            po = w.pod_off[: n + 1]
            claims = w.claims[: int(po[-1])]
            prio = w.prio[:n]
            flags = pkg.api.F_EXHAUSTIVE if it % 2 else 0
            cands = None if it % 3 == 0 else _cands(rng, n, _nn(w), 1 + it)
            mv = (0, 3, 16)[it % 3]
            ref = _oracle(pkg, W.state(), w, claims, po, prio, cands, mv, flags)
            for r, got in enumerate(W.call(claims, po, prio, run, cands, mv, flags, pairs=it % 2 == 0)):
                _same(got, ref, f"call {it} rank {r}", pairs=it % 2 == 0)
            # sharded UnsuitableNodes on the same buffer
            d_c, d_p = _dev(claims), _dev(po)
            bits = [torch.zeros(((n * _nn(w) + 7) // 8 + 16,), dtype=torch.uint8, device="cuda:0") for _ in W.ctxs]
            torch.cuda.synchronize()
            for c, b in zip(W.ctxs, bits):
                c.unsuitable_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n, None, None, n * _nn(w),
                                           b.data_ptr(), flags)
            for c in W.ctxs:
                c.sync()
            assert all(b.cpu().numpy().tobytes() == bits[0].cpu().numpy().tobytes() for b in bits)
            # pods Allocate of a few pending pods onto their first candidate's node, then the inventory sync
            pod = w.claims[w.pod_off[it]: w.pod_off[it + 1]].copy()
            pod["node"] = (it * 5) % _nn(w)
            oo, n_out = R.out_offsets(pod, _nn(w))
            d_pod, d_ppo, d_oo = _dev(pod), _dev(np.array([0, len(pod)], np.uint32)), _dev(oo)
            torch.cuda.synchronize()
            for c in W.ctxs:
                c.allocate_pods_global_device(d_pod.data_ptr(), len(pod), d_ppo.data_ptr(), 1, d_oo.data_ptr(), n_out, 0)
            for c in W.ctxs:
                c.shard_sync_inventory_device()
            for c in W.ctxs:
                c.sync()
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
    W = World(pkg, w, world, _bounds(_nn(w), world, "uneven"))
    try:
        po, cands = w.pod_off.copy(), None
        rc, rpo, rpr, ro = w.run_claims, w.run_pod_off, w.run_prio, w.run_out
        if kind == "pod_off":
            po[5] = po[6] + 1
        elif kind == "cand_off":
            cn, co = _cands(np.random.default_rng(0), len(po) - 1, _nn(w), 4)
            co[3] = co[4] + 2
            cands = (cn, co)
        else:
            rc, rpo, rpr, ro = _bad_running(w, kind)
        run = Running(pkg, rc, rpo, rpr, ro)
        outs, meta = W.enqueue(w.claims, po, w.prio, run, cands, 16, 0)
        for r, c in enumerate(W.ctxs):
            with pytest.raises(A.DraError) as e:
                c.sync()
            assert e.value.code == A.E_INVAL, (kind, r)
        for r, o in enumerate(outs):
            assert all((t.cpu().numpy() == SENTINEL).all() for t in o), f"{kind}: rank {r} wrote an output"
        # the next valid call on the same world matches the oracle
        _check_all(pkg, W, w, _running(pkg, w), [(0, "cands", 16, True)], np.random.default_rng(2), f"after {kind}")
    finally:
        W.close()


def test_host_side_errors(pkg):
    A = pkg.api
    w = pkg.synth.preempt(n_node=12, gpus_per_node=8, n_pending=20, seed=5)
    n_pod = len(w.pod_off) - 1
    W = World(pkg, w, 2, _bounds(_nn(w), 2, "even"), sizes=(n_pod, n_pod * _nn(w), 8))
    try:
        run = _running(pkg, w)
        c = W.ctxs[0]
        import torch
        keep = [_dev(w.claims), _dev(w.pod_off), _dev(w.prio)]
        o = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda:0").data_ptr()
        n_pair = n_pod * _nn(w)
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
    W = World(pkg, w, 2, _bounds(_nn(w), 2, "even"), sizes=(n_pod - 1, n_pod * _nn(w), 8))
    try:
        with pytest.raises(A.DraError) as e:
            W.enqueue(w.claims, w.pod_off, w.prio, _running(pkg, w), None, 8)
        assert e.value.code == A.E_INVAL
    finally:
        W.close()
    # a bare dra_set_shard, and a world with no export
    for kw in (dict(bare=True), dict(export=False)):
        W = World(pkg, w, 2, _bounds(_nn(w), 2, "even"), **kw)
        try:
            with pytest.raises(A.DraError) as e:
                W.enqueue(w.claims, w.pod_off, w.prio, _running(pkg, w), None, 8)
            assert e.value.code == A.E_STATE, kw
        finally:
            W.close()


def test_multi_process_preempt():
    """tests/multi_gpu_shard_preempt_check.py under torchrun: one process per GPU, peers mapped with IPC handles."""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = min(n, 4)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", "29643",
                        os.path.join(ROOT, "tests", "multi_gpu_shard_preempt_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
