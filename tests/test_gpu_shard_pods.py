"""GPU suite: pods Allocate on a sharded world (dra_allocate_pods_batch_global_device).  World contexts of this process on
ONE device, wired with dra_comm_init_local / dra_peer_import_local like test_gpu_shard_unsuitable.py.  Every rank's whole
table must be byte for byte the oracle's answer on the world's real state (the inventory each rank holds for its own node
range), each rank's own GPU range the oracle's inventory afterwards, and no rank may write GPUs outside its range."""
import os

import numpy as np
import pytest

from test_gpu_shard_unsuitable import _bounds, _dense, _dev, _pod_cuts

pytestmark = pytest.mark.gpu

N_OUT_MAX = 1 << 16


class PodWorld:
    """world contexts on device 0, every one holding the whole inventory, rank r serving [bounds[r], bounds[r+1])."""

    def __init__(self, pkg, w, world, bounds, stray_rank=0, max_pairs=0, attrs=None, sels=None, cap_per_rank=0):
        R = pkg.records
        self.pkg, self.w, self.world, self.bounds = pkg, w, world, list(bounds)
        self.ctxs = [pkg.api.Context(device=0) for _ in range(world)]
        for r, c in enumerate(self.ctxs):
            c.comm_init_local(r, world)
            c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
            if sels is not None:
                c.set_gpu_attrs(attrs); c.set_selectors(sels.reshape(-1, R.SEL_MAX_INS))
            c.set_shard_map(bounds, stray_rank=stray_rank)
            if world > 1:
                if max_pairs:
                    c.set_shard_pairs(max_pairs)
                c.shard_export(N_OUT_MAX, cap_per_rank, want_handle=False)
        if world > 1:
            for c in self.ctxs:
                c.peer_import_local(self.ctxs)

    def close(self):
        for c in self.ctxs:
            c.close()

    def gpu_range(self, r):
        off = self.w.node_off
        return int(off[self.bounds[r]]), int(off[self.bounds[r + 1]])

    def inventories(self):
        return [c.get_inventory() for c in self.ctxs]

    def real_state(self):
        """The world's state: every rank's copy over its own GPU range."""
        real = self.w.gpus.copy()
        for r, inv in enumerate(self.inventories()):
            g0, g1 = self.gpu_range(r)
            real[g0:g1] = inv[g0:g1]
        return real

    def enqueue(self, claims, pod_off, out_off, n_out, flags=0):
        import torch
        keep = [_dev(claims) if len(claims) else torch.zeros(16, dtype=torch.uint8, device="cuda:0"), _dev(pod_off),
                _dev(out_off) if out_off is not None else None]
        torch.cuda.synchronize()                         # (the contexts' streams do not wait for torch's)
        for c in self.ctxs:
            c.allocate_pods_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), len(pod_off) - 1,
                                          keep[2].data_ptr() if keep[2] is not None else None, n_out, flags)
        return keep

    def call(self, claims, pod_off, out_off, n_out, flags=0):
        """The call on every rank (enqueued on all of them first, then waited for); every rank's whole table."""
        keep = self.enqueue(claims, pod_off, out_off, n_out, flags)
        for c in self.ctxs:
            c.sync()
        del keep
        return [c.gather_read(np.zeros(n_out, dtype=self.pkg.records.OUT_DTYPE)) for c in self.ctxs]

    def check(self, oracle, claims, pod_off, out_off, n_out, flags, what):
        """One call against the oracle on the real state (the pristine inventory under F_FRESH_INVENTORY)."""
        api = self.pkg.api
        before = self.inventories()
        src = self.w.gpus if flags & api.F_FRESH_INVENTORY else self.real_state()
        oflags = oracle.F_EXHAUSTIVE if flags & api.F_EXHAUSTIVE else 0
        ref, ref_inv = oracle.allocate_pods(src, self.w.node_off, self.w.table, claims, pod_off, out_off, n_out, oflags)
        tables = self.call(claims, pod_off, out_off, n_out, flags)
        after = self.inventories()
        for r in range(self.world):
            assert tables[r].tobytes() == ref.tobytes(), f"{what}: rank {r} table differs"
            g0, g1 = self.gpu_range(r)
            assert after[r][g0:g1].tobytes() == ref_inv[g0:g1].tobytes(), f"{what}: rank {r} inventory of its range differs"
            assert after[r][:g0].tobytes() == before[r][:g0].tobytes() and \
                after[r][g1:].tobytes() == before[r][g1:].tobytes(), f"{what}: rank {r} wrote GPUs outside its range"
        return ref


def _flags(api):
    return [0, api.F_EXHAUSTIVE, api.F_FRESH_INVENTORY, api.F_EXHAUSTIVE | api.F_FRESH_INVENTORY]


def _malformed_mixed(pkg, w, bounds, rng, with_off):
    """Pods cut from synth.mixed, most on one node, plus pods shaped to hit the ownership rule: a GPU claim with count > 1
    naming another rank's node inside a mixed-node pod, a first claim naming no node before valid ones, a pod of more
    than 32 claims spanning ranks, empty pods and pods on the nodes at range boundaries."""
    R = pkg.records
    claims = w.claims.copy()
    pod_off = _pod_cuts(rng, w.n_claim, 500, big=True)
    n_pod, n_node = len(pod_off) - 1, w.n_node
    for p in range(n_pod):
        if rng.integers(0, 10):
            claims["node"][pod_off[p]: pod_off[p + 1]] = claims["node"][pod_off[p]]
    sizes = np.diff(pod_off.astype(np.int64))
    multi = [p for p in range(n_pod) if 2 <= sizes[p] <= 32]
    edges = sorted({b for b in bounds if 0 < b < n_node} | {b - 1 for b in bounds if 0 < b <= n_node})
    for k, p in enumerate(multi[:len(edges)]):           # pods exactly at the range boundaries
        claims["node"][pod_off[p]: pod_off[p + 1]] = edges[k]
    rest = multi[len(edges):]
    p = rest[0]                                          # GPU count 3 on another rank's node inside a mixed-node pod
    i = pod_off[p] + 1
    first = int(claims["node"][pod_off[p]])
    claims["node"][i] = (first + n_node // 2 + 1) % n_node
    claims["kind"][i], claims["count"][i], claims["profile"][i] = R.KIND_GPU, 3, 0
    p = rest[1]                                          # first claim names no node, the later ones valid nodes
    claims["node"][pod_off[p]] = n_node + 5
    claims["node"][pod_off[p] + 1: pod_off[p + 1]] = rng.integers(0, n_node, sizes[p] - 1)
    big = int(np.argmax(sizes))                          # the pod of > 32 claims spans every rank's nodes
    assert sizes[big] > 32
    claims["node"][pod_off[big]: pod_off[big + 1]] = np.arange(sizes[big]) % n_node
    if with_off:
        out_off, n_out = R.out_offsets(claims, n_node)
        return claims, pod_off, out_off, int(n_out)
    return claims, pod_off, None, len(claims)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("workload", ["pods", "mixed_off", "mixed_nooff"])
def test_matches_oracle(pkg, oracle, world, workload):
    """Every flag combination, one after the other on the same world; every rank's whole table and own range checked."""
    api = pkg.api
    rng = np.random.default_rng(world * 7 + len(workload))
    kind = ["even", "uneven", "empty", "even"][world - 1] if world > 1 else "even"
    stray = world - 1                                    # stray_rank != 0 from world 2 on
    attrs = sels = None
    if workload == "pods":
        w, pod_off = pkg.synth.pods(700, 29, world)
        bounds = _bounds(w.n_node, world, kind)
        jobs = [(w.claims, pod_off, None, w.n_claim)]
    else:
        w = pkg.synth.mixed(2400, 31, 60 + world, invalid=True)
        attrs, sels = pkg.synth.with_selectors(w, world)
        bounds = _bounds(w.n_node, world, kind)
        jobs = [_malformed_mixed(pkg, w, bounds, rng, workload == "mixed_off")]
    W = PodWorld(pkg, w, world, bounds, stray, attrs=attrs, sels=sels)
    oracle.set_selectors(attrs, sels)
    try:
        for flags in _flags(api):
            for claims, po, oo, n_out in jobs:
                ref = W.check(oracle, claims, po, oo, n_out, flags, f"{workload} flags {flags}")
                st = ref["status"]
                if flags in (0, api.F_FRESH_INVENTORY):
                    assert (st == pkg.records.ST_OK).any() and (st == pkg.records.ST_POD).any()
                if workload != "pods":
                    assert (st == pkg.records.ST_INVALID).any()
        if workload == "pods":
            ff = oracle.allocate_pods(w.gpus, w.node_off, w.table, w.claims, pod_off)[0]
            ex = oracle.allocate_pods(w.gpus, w.node_off, w.table, w.claims, pod_off, flags=oracle.F_EXHAUSTIVE)[0]
            assert ff.tobytes() != ex.tobytes(), "the workload does not separate first-fit from the exhaustive search"
    finally:
        oracle.set_selectors()
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_allocate_then_pods(pkg, oracle, world):
    """The gap the call closes: after a sharded Allocate without F_FRESH_INVENTORY each rank's copy is right for its own
    nodes only.  dra_allocate_pods_batch on rank 0 answers from its stale copy; the sharded call answers on the real state."""
    R = pkg.records
    w, pod_off = pkg.synth.pods(900, 32, 40 + world)
    bounds = _bounds(w.n_node, world, "even")
    W = PodWorld(pkg, w, world, bounds, 0)
    try:
        half = int(pod_off[450])
        d = _dev(w.claims[:half])
        for c in W.ctxs:
            c.allocate_global_device(d.data_ptr(), half, None, half, 0)
        for c in W.ctxs:
            c.gather_read(np.zeros(half, dtype=R.OUT_DTYPE))
        real = W.real_state()
        _, ref_real = oracle.allocate(w.gpus, w.node_off, w.table, w.claims[:half])
        assert real.tobytes() == ref_real.tobytes()
        claims, po = w.claims[half:], (pod_off[450:] - half).astype(np.uint32)
        ref = oracle.allocate_pods(real, w.node_off, w.table, claims, po, flags=oracle.F_EXHAUSTIVE)[0]
        stale = W.ctxs[0].allocate_pods(claims, po, flags=pkg.api.F_EXHAUSTIVE)
        assert stale.tobytes() != ref.tobytes(), "the workload does not expose the stale copies"
        W.check(oracle, claims, po, None, len(claims), pkg.api.F_EXHAUSTIVE, "after a sharded allocate")
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 4])
def test_world_acts_on_its_own_verdict(pkg, oracle, world):
    """Sharded Allocate -> sharded exhaustive UnsuitableNodes -> for each pod a suitable node (one pod per node), claims
    retargeted there -> the sharded pods Allocate with F_EXHAUSTIVE places every one of those pods."""
    import torch
    R, api = pkg.records, pkg.api
    w, pod_off = pkg.synth.pods(500, 40, 70 + world)
    bounds = _bounds(w.n_node, world, "uneven")
    first = int(pod_off[200])
    n_pod = 300
    W = PodWorld(pkg, w, world, bounds, world - 1, max_pairs=n_pod * w.n_node)
    try:
        d = _dev(w.claims[:first])
        for c in W.ctxs:
            c.allocate_global_device(d.data_ptr(), first, None, first, 0)
        for c in W.ctxs:
            c.gather_read(np.zeros(first, dtype=R.OUT_DTYPE))
        claims = w.claims[first:].copy()
        po = (pod_off[200:] - first).astype(np.uint32)
        d_c, d_p = _dev(claims), _dev(po)
        n_pair = n_pod * w.n_node
        bits = [torch.zeros((n_pair + 7) // 8 + 8, dtype=torch.uint8, device="cuda:0") for _ in W.ctxs]
        torch.cuda.synchronize()
        for c, b in zip(W.ctxs, bits):
            c.unsuitable_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n_pod, None, None, n_pair, b.data_ptr(),
                                       api.F_EXHAUSTIVE)
        for c in W.ctxs:
            c.sync()
        verdict = [np.unpackbits(b.cpu().numpy()[: (n_pair + 7) // 8], bitorder="little")[:n_pair].reshape(n_pod, w.n_node)
                   for b in bits]
        for v in verdict[1:]:
            assert (v == verdict[0]).all()
        real = W.real_state()
        dn, do = _dense(n_pod, w.n_node)
        ref_bits = oracle.unsuitable(real, w.node_off, w.table, claims, po, dn, do, flags=oracle.F_EXHAUSTIVE)
        assert np.packbits(verdict[0].ravel(), bitorder="little").tobytes() == ref_bits.tobytes()
        taken, keep = set(), []
        for p in range(n_pod):
            free = [n for n in np.flatnonzero(verdict[0][p]) if n not in taken]
            if free:
                n = int(free[len(free) // 2]); taken.add(n)
                keep.append((p, n))
        assert len(keep) >= 10
        sel = np.concatenate([np.arange(po[p], po[p + 1]) for p, _ in keep])
        sub = claims[sel].copy()
        sub_off = np.zeros(len(keep) + 1, dtype=np.uint32)
        sub_off[1:] = np.cumsum([po[p + 1] - po[p] for p, _ in keep])
        for k, (_, n) in enumerate(keep):
            sub["node"][sub_off[k]: sub_off[k + 1]] = n
        ref = W.check(oracle, sub, sub_off, None, len(sub), api.F_EXHAUSTIVE, "pods on their suitable nodes")
        assert (ref["status"] == 0).all(), "a pod the exhaustive verdict called suitable was not placed"
    finally:
        W.close()


def test_world1_equals_single_inventory_call(pkg, oracle):
    """World 1 over [0, n_node): OutRecs and inventory byte for byte those of dra_allocate_pods_batch, every flag."""
    R, api = pkg.records, pkg.api
    w = pkg.synth.mixed(2000, 29, 88, invalid=True)
    claims, pod_off, out_off, n_out = _malformed_mixed(pkg, w, [0, w.n_node], np.random.default_rng(9), True)
    W = PodWorld(pkg, w, 1, [0, w.n_node], 0)
    with api.Context(device=0) as single:
        single.set_table(w.table); single.set_inventory(w.gpus, w.node_off)
        try:
            for flags in _flags(api):
                got = W.call(claims, pod_off, out_off, n_out, flags)[0]
                ref = single.allocate_pods(claims, pod_off, out_off, n_out, flags)
                assert got.tobytes() == ref.tobytes(), f"flags {flags}"
                assert W.ctxs[0].get_inventory().tobytes() == single.get_inventory().tobytes(), f"flags {flags}"
            assert W.ctxs[0].last_chain() >= {"pod_shard"} and "pod_gather" not in W.ctxs[0].last_chain()
        finally:
            W.close()


def test_consecutive_calls_interleaved(pkg, oracle):
    """Pods calls of changing size between sharded Allocates and sharded UnsuitableNodes on the same export: the epoch
    parity, the packet cursors and the peer buffer shared by the three calls."""
    import torch
    R, api = pkg.records, pkg.api
    world = 3
    w, pod_off = pkg.synth.pods(3000, 30, 5)
    bounds = _bounds(w.n_node, world, "uneven")
    W = PodWorld(pkg, w, world, bounds, 1, max_pairs=400 * w.n_node)
    rng = np.random.default_rng(4)
    try:
        for step, n_pod in enumerate([400, 1, 37, 211, 3, 150, 64]):
            if step % 2 == 0:                            # a sharded allocate of a slice of the claims
                lo = int(pod_off[step * 200])
                part = w.claims[lo: lo + 300]
                dp = _dev(part)
                for c in W.ctxs:
                    c.allocate_global_device(dp.data_ptr(), len(part), None, len(part), 0)
                for c in W.ctxs:
                    c.gather_read(np.zeros(len(part), dtype=R.OUT_DTYPE))
            p0 = int(rng.integers(0, 3000 - n_pod))
            claims = w.claims[pod_off[p0]: pod_off[p0 + n_pod]]
            po = (pod_off[p0: p0 + n_pod + 1] - pod_off[p0]).astype(np.uint32)
            if step % 3 == 1:                            # a sharded exhaustive UnsuitableNodes in between
                n_pair = n_pod * w.n_node
                d_c, d_p = _dev(claims), _dev(po)
                bits = [torch.zeros((n_pair + 7) // 8 + 8, dtype=torch.uint8, device="cuda:0") for _ in W.ctxs]
                torch.cuda.synchronize()
                for c, b in zip(W.ctxs, bits):
                    c.unsuitable_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n_pod, None, None, n_pair,
                                               b.data_ptr(), api.F_EXHAUSTIVE)
                for c in W.ctxs:
                    c.sync()
                dn, do = _dense(n_pod, w.n_node)
                ref = oracle.unsuitable(W.real_state(), w.node_off, w.table, claims, po, dn, do, flags=oracle.F_EXHAUSTIVE)
                for r, b in enumerate(bits):
                    assert b.cpu().numpy()[: len(ref)].tobytes() == ref.tobytes(), f"step {step} rank {r} bits"
            flags = api.F_EXHAUSTIVE if step % 2 else 0
            W.check(oracle, claims, po, None, len(claims), flags, f"step {step}")
        assert W.ctxs[0].last_chain() >= {"pod_shard", "pod_gather"}
    finally:
        W.close()


def test_errors(pkg, oracle):
    """Host-side checks return before anything is enqueued.  Device-side faults (pod_off not monotone or short, slots past
    n_out, a rank owning more slots than its packet room) give DRA_E_INVAL on EVERY rank with no inventory changed, and the
    next valid call is right."""
    import torch
    R, api = pkg.records, pkg.api
    w = pkg.synth.mixed(600, 11, 3, invalid=True)
    bounds = [0, 5, 11]
    pod_off = np.arange(0, 61, 3, dtype=np.uint32)
    claims = w.claims[: pod_off[-1]].copy()
    for p in range(20):
        claims["node"][pod_off[p]: pod_off[p + 1]] = claims["node"][pod_off[p]]
    out_off, n_out = R.out_offsets(claims, w.n_node)
    n_out = int(n_out)
    d_c, d_p, d_o = _dev(claims), _dev(pod_off), _dev(out_off)
    torch.cuda.synchronize()

    def raw(c, **k):
        a = dict(claims=d_c.data_ptr(), n_claim=len(claims), pod_off=d_p.data_ptr(), n_pod=20, out_off=d_o.data_ptr(),
                 n_out=n_out, flags=0)
        a.update(k)
        return c._lib.dra_allocate_pods_batch_global_device(c._h, a["claims"], a["n_claim"], a["pod_off"], a["n_pod"],
                                                            a["out_off"], a["n_out"], a["flags"])

    with api.Context(device=0) as c:
        c.set_table(w.table); c.set_inventory(w.gpus, w.node_off)
        assert raw(c) == api.E_STATE                                         # no shard
        c.comm_init_local(0, 2); c.set_shard(0, 5, take_stray=True)
        assert raw(c) == api.E_STATE                                         # world 2 after a bare set_shard
        c.set_shard_map(bounds, 0)
        assert raw(c) == api.E_STATE                                         # world 2 without export + import
    W = PodWorld(pkg, w, 2, bounds, 1)
    try:
        c0 = W.ctxs[0]
        assert raw(c0, flags=0x80) == api.E_INVAL                            # unknown flag
        assert raw(c0, flags=api.F_NODE_SORTED) == api.E_INVAL
        assert raw(c0, n_out=N_OUT_MAX + 1) == api.E_INVAL                   # past the exported table
        assert raw(c0, out_off=None, n_out=len(claims) - 1) == api.E_INVAL   # n_out < n_claim without out_off
        assert raw(c0, n_pod=0) == api.E_INVAL                               # claims but no pods
        assert raw(c0, n_claim=(1 << 26) + 1) == api.E_INVAL
        W.check(oracle, claims, pod_off, out_off, n_out, 0, "after host-side errors")
        bad_po = pod_off.copy(); bad_po[5] = bad_po[7] + 1
        short_po = pod_off.copy(); short_po[-1] -= 1
        past = out_off.copy(); past[-1] = n_out
        for po, oo, flags in ((bad_po, out_off, 0), (short_po, out_off, api.F_FRESH_INVENTORY), (pod_off, past, api.F_EXHAUSTIVE)):
            before = W.inventories()
            keep = W.enqueue(claims, po, oo, n_out, flags)
            codes = []
            for c in W.ctxs:
                try:
                    c.sync(); codes.append(0)
                except api.DraError as e:
                    codes.append(e.code)
            del keep
            assert codes == [api.E_INVAL] * 2, codes
            for b, a in zip(before, W.inventories()):
                assert a.tobytes() == b.tobytes(), "a failed call changed an inventory"
            W.check(oracle, claims, pod_off, out_off, n_out, api.F_EXHAUSTIVE, "after a device-side error")
    finally:
        W.close()
    # more slots on one rank than the packet room its export reserved: every rank fails, nothing changes
    W = PodWorld(pkg, w, 2, bounds, 1, cap_per_rank=8)
    try:
        before = W.inventories()
        keep = W.enqueue(claims, pod_off, out_off, n_out, 0)
        codes = []
        for c in W.ctxs:
            try:
                c.sync(); codes.append(0)
            except api.DraError as e:
                codes.append(e.code)
        del keep
        assert codes == [api.E_INVAL] * 2, codes
        for b, a in zip(before, W.inventories()):
            assert a.tobytes() == b.tobytes()
        # two pods without out_off (one slot per claim): within the room
        W.check(oracle, claims[:6], pod_off[:3], None, 6, 0, "within the packet room")
    finally:
        W.close()


def test_empty_and_zero_shapes(pkg, oracle):
    """Only empty pods, n_pod == 0, one pod of one claim on the last node, and a world with an empty range."""
    w = pkg.synth.mixed(400, 13, 12, invalid=True)
    world = 4
    W = PodWorld(pkg, w, world, _bounds(w.n_node, world, "empty"), 2)
    try:
        z = _dev(np.zeros(4, dtype=np.uint32))
        for c in W.ctxs:
            c.allocate_pods_global_device(0, 0, z.data_ptr(), 0, None, 0, 0)
        for c in W.ctxs:
            c.sync()
        one = w.claims[:1].copy(); one["node"] = w.n_node - 1
        W.check(oracle, one, np.array([0, 1], dtype=np.uint32), None, 1, 0, "one pod")
        W.check(oracle, w.claims[:0], np.zeros(4, dtype=np.uint32), None, 1, 0, "only empty pods")
        po = np.array([0, 0, 5, 5, 9, 9], dtype=np.uint32)
        c = w.claims[:9].copy(); c["node"][:5] = 0; c["node"][5:] = w.n_node - 1
        W.check(oracle, c, po, None, 9, pkg.api.F_EXHAUSTIVE, "empty pods between")
    finally:
        W.close()


@pytest.mark.parametrize("world", [2, 3])
def test_pod_problems_replayed_sharded(pkg, oracle, world):
    """The pod-mode property generator through the sharded call with random bounds and stray rank."""
    from hypothesis import HealthCheck, given, settings
    from hypothesis import strategies as st
    from test_pod_mode import pod_problems
    R, api = pkg.records, pkg.api
    n_ex = int(os.environ.get("DRA_PROP_EXAMPLES", "0"))
    ctxs = [api.Context(device=0) for _ in range(world)]
    try:
        for r, c in enumerate(ctxs):
            c.comm_init_local(r, world)
            c.shard_export(4096, 0, want_handle=False)
        for c in ctxs:
            c.peer_import_local(ctxs)

        @settings(max_examples=n_ex or 80, deadline=None, suppress_health_check=list(HealthCheck), derandomize=n_ex == 0,
                  database=None)
        @given(pod_problems(), st.booleans(), st.booleans(), st.data())
        def run(prob, exhaustive, fresh, data):
            g, off, t, c, pod_off, out_off, n_out = prob
            n_node = len(off) - 1
            cuts = sorted(data.draw(st.lists(st.integers(0, n_node), min_size=world - 1, max_size=world - 1)))
            bounds = [0] + cuts + [n_node]
            stray = data.draw(st.integers(0, world - 1))
            for x in ctxs:
                x.set_table(t); x.set_inventory(g, off); x.set_shard_map(bounds, stray_rank=stray)
            w = type("W", (), {})()
            w.gpus, w.node_off, w.table = g, off, t
            W = PodWorld.__new__(PodWorld)
            W.pkg, W.w, W.world, W.bounds, W.ctxs = pkg, w, world, bounds, ctxs
            flags = (api.F_EXHAUSTIVE if exhaustive else 0) | (api.F_FRESH_INVENTORY if fresh else 0)
            n_out = max(int(n_out), 1)
            if len(pod_off) - 1 == 0:
                return
            W.check(oracle, c, pod_off, out_off, n_out, flags, f"bounds {bounds} stray {stray}")

        run()
    finally:
        for c in ctxs:
            c.close()
