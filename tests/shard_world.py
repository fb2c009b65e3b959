"""The sharded world of the single-device GPU suites (tests/test_gpu_shard*.py): world contexts of this process on ONE
device, each with its own stream, wired with dra_comm_init_local / dra_peer_import_local (the form a single driver
process uses; torchrun ranks use IPC handles instead: tests/multi_gpu_rank.py).  One function per sharded call runs it on
every rank, enqueued on all of them before any waits, and reads every rank's outputs back.  Not collected by pytest."""
import ctypes as C

import numpy as np

NONE = 0xFFFFFFFF
PAD = 16                                                 # sentinel bytes past every output


def dev(a):
    """a's bytes on cuda:0; 16 zero bytes for an empty array, so the pointer is never null."""
    import torch
    a = np.ascontiguousarray(a)
    if a.nbytes == 0:
        return torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to("cuda:0")


def ptr(t):
    return None if t is None else t.data_ptr()


def nn(w):
    return len(w.node_off) - 1


def bounds(n_node, world, kind):
    if kind == "even":
        return [n_node * r // world for r in range(world)] + [n_node]
    if kind == "uneven":                                  # rank 0 a sliver, the last rank most of it
        b = [0] + [min(n_node, 1 + 2 * r * r) for r in range(1, world)] + [n_node]
        return sorted(b)
    # "empty": an empty range in the middle and one at the end
    b = [0] + [n_node // 2] * (world - 1) + [n_node]
    if world > 2:
        b[-2] = n_node
    return b


def dense(n_pod, n_node):
    """The dense form's pairs as candidate lists: every node for every pod."""
    return (np.tile(np.arange(n_node, dtype=np.uint32), n_pod),
            (np.arange(n_pod + 1, dtype=np.uint64) * n_node).astype(np.uint32))


def cands(rng, n_pod, n_node, k):
    """k candidates per pod, duplicates and nodes past the inventory included."""
    nodes = rng.integers(0, n_node + 3, size=n_pod * k).astype(np.uint32)
    if len(nodes) > 3:
        nodes[1] = nodes[0]
        nodes[2] = NONE
    return nodes, (np.arange(n_pod + 1) * k).astype(np.uint32)


def candidates(rng, n_pod, n_node):
    """0-8 candidates per pod, every seventh pod none, some naming no node, a repeated one and NONE."""
    per = rng.integers(0, 9, n_pod)
    per[::7] = 0
    cand_off = np.zeros(n_pod + 1, dtype=np.uint32); cand_off[1:] = np.cumsum(per)
    cand_nodes = rng.integers(0, n_node + 4, int(cand_off[-1])).astype(np.uint32)
    if len(cand_nodes) > 3:
        cand_nodes[1] = cand_nodes[0]
        cand_nodes[2] = NONE
    return cand_nodes, cand_off


def pod_cuts(rng, n_claim, n_cut, big=False):
    cuts = np.unique(np.concatenate([[0, n_claim], rng.integers(0, n_claim, n_cut)])).astype(np.uint32)
    cuts = np.insert(cuts, 3, cuts[3])                   # an empty pod
    if big and n_claim > 100:
        cuts = np.unique(np.concatenate([cuts[cuts < 40], cuts[cuts > 80]])).astype(np.uint32)   # one pod of > 32 claims
        cuts = np.insert(cuts, 1, cuts[1])
    return cuts


def malformed_mixed(pkg, w, bounds, rng, with_off):
    """Pods cut from synth.mixed, most on one node, plus pods shaped to hit the ownership rule: a GPU claim with count > 1
    naming another rank's node inside a mixed-node pod, a first claim naming no node before valid ones, a pod of more
    than 32 claims spanning ranks, empty pods and pods on the nodes at range boundaries."""
    R = pkg.records
    claims = w.claims.copy()
    pod_off = pod_cuts(rng, w.n_claim, 500, big=True)
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


def shared_mixed(pkg, w, rng):
    """synth.mixed's claims with a fifth of them turned into cfg4-style SHARED claims (MPS limits of 1-10 GiB)."""
    R = pkg.records
    c = w.claims.copy()
    sh = rng.random(len(c)) < 0.2
    c["kind"][sh], c["count"][sh], c["group"][sh] = R.KIND_SHARED, 1, 0
    c["mem_limit_mib"][sh] = rng.choice(np.array([1024, 2048, 4096, 8192, 10240], dtype=np.uint32), int(sh.sum()))
    return c


class Running:
    """The running pods on the device, and the dra_running_pods struct pointing at them."""

    def __init__(self, pkg, claims, pod_off, prio, out, out_off=None, out_ptr=None):
        self.keep = [dev(claims), dev(pod_off), dev(prio), dev(out)] + ([dev(out_off)] if out_off is not None else [])
        self.struct = pkg.api.RunningPods(self.keep[0].data_ptr(), len(claims), self.keep[1].data_ptr(), len(pod_off) - 1,
                                          self.keep[2].data_ptr(), self.keep[4].data_ptr() if out_off is not None else None,
                                          out_ptr if out_ptr is not None else self.keep[3].data_ptr(), len(out))


def table_ptr(c):
    """Device pointer of the context's last gathered table (dra_gather_table)."""
    p, n = C.c_void_p(), C.c_uint32()
    rc = c._lib.dra_gather_table(c._h, C.byref(p), C.byref(n))
    assert rc == 0, rc
    return p.value


def same(got, ref, names, what):
    """Each output byte for byte the oracle's; an output that is None (not asked for) is skipped."""
    for name, x, y in zip(names, got, ref):
        if x is not None and x.tobytes() != y.tobytes():
            bad = np.flatnonzero(x.reshape(-1) != y.reshape(-1))[:5]
            raise AssertionError(f"{what}: {name} differs at {bad}: device {x.reshape(-1)[bad]} oracle {y.reshape(-1)[bad]}")


def same_tables(tables, ref, what):
    for r, t in enumerate(tables):
        assert t.tobytes() == ref.tobytes(), f"{what}: rank {r} table differs from the oracle"


class World:
    """world contexts on device 0, rank r serving [bounds[r], bounds[r+1]) of the inventory it was given: `inv` is one
    inventory for every rank or a list of one per rank.  The ranks' ranges come from dra_set_shard_map, or from a bare
    dra_set_shard each (bare=True); bounds None sets no shard at all.  Each size keyword is one dra_set_shard_<name> call,
    made before the export (a size only takes effect at the export); a world of 1 neither exports nor imports, nor does
    one built with export=False."""

    def __init__(self, pkg, table, node_off, inv, world, bounds, stray_rank=0, attrs=None, sels=None, bare=False, export=True,
                 n_out_max=64, cap_per_rank=0, pairs=None, place=None, preempt=None, capacity=None, preempt_place=None):
        R = pkg.records
        self.pkg, self.table, self.node_off, self.world = pkg, table, node_off, world
        self.bounds = None if bounds is None else list(bounds)
        self.n_node = len(node_off) - 1
        self.loaded = list(inv) if isinstance(inv, (list, tuple)) else [inv] * world
        self.ctxs = [pkg.api.Context(device=0) for _ in range(world)]
        for r, c in enumerate(self.ctxs):
            c.comm_init_local(r, world)
            c.set_table(table); c.set_inventory(self.loaded[r], node_off)
            if sels is not None:
                c.set_gpu_attrs(attrs); c.set_selectors(sels.reshape(-1, R.SEL_MAX_INS))
            if bounds is None:
                pass
            elif bare:
                c.set_shard(bounds[r], bounds[r + 1], take_stray=r == stray_rank)
            else:
                c.set_shard_map(bounds, stray_rank=stray_rank)
            if pairs is not None:
                c.set_shard_pairs(pairs)
            if place is not None:
                c.set_shard_place(place)
            if preempt is not None:
                c.set_shard_preempt(*preempt)
            if capacity is not None:
                c.set_shard_capacity(capacity)
            if preempt_place is not None:
                c.set_shard_preempt_place(*preempt_place)
            if world > 1 and export:
                c.shard_export(n_out_max, cap_per_rank, want_handle=False)
        if world > 1 and export:
            for c in self.ctxs:
                c.peer_import_local(self.ctxs)

    def close(self):
        for c in self.ctxs:
            c.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def gpu_range(self, r):
        return int(self.node_off[self.bounds[r]]), int(self.node_off[self.bounds[r + 1]])

    def inventories(self):
        return [c.get_inventory() for c in self.ctxs]

    def state(self):
        """The world's state: every rank's copy over its own GPU range."""
        g = self.loaded[0].copy()
        for r, inv in enumerate(self.inventories()):
            a, b = self.gpu_range(r)
            g[a:b] = inv[a:b]
        return g

    def each(self, fn, expect=0):
        """fn(r, ctx) enqueued on every rank first, then every rank waited for: each must end with the code `expect`."""
        import torch
        torch.cuda.synchronize()                         # (the contexts' streams do not wait for torch's uploads)
        for r, c in enumerate(self.ctxs):
            fn(r, c)
        self.wait(expect)

    def wait(self, expect=0):
        """Every rank waited for, with no device-wide wait before: each must end with the code `expect`."""
        codes = []
        for c in self.ctxs:
            try:
                c.sync(); codes.append(0)
            except self.pkg.api.DraError as e:
                codes.append(e.code)
        assert codes == [expect] * self.world, codes

    def sync_inventory(self):
        """The inventory sync enqueued on every rank behind whatever the ranks' streams already hold, then waited for."""
        for c in self.ctxs:
            c.shard_sync_inventory_device()
        self.wait()

    def remap(self, bounds, stray_rank):
        for c in self.ctxs:
            c.set_shard_map(bounds, stray_rank=stray_rank)
        self.bounds = list(bounds)

    def outputs(self, sizes, sentinel):
        """One sentinel-filled device buffer per output size, PAD bytes longer, for every rank."""
        import torch
        return [[torch.full((s + PAD,), sentinel, dtype=torch.uint8, device="cuda:0") for s in sizes] for _ in self.ctxs]

    def read(self, outs, sizes, dtypes, names, asked, sentinel):
        """Every rank's outputs as arrays, None where not asked for.  Nothing may be written past an output, nor into one
        that was not asked for."""
        res = []
        for r, o in enumerate(outs):
            got = []
            for t, s, d, name, a in zip(o, sizes, dtypes, names, asked):
                h = t.cpu().numpy()
                assert (h[s:] == sentinel).all(), f"rank {r} wrote past {name}"
                if not a:
                    assert (h == sentinel).all(), f"rank {r} wrote {name} without being asked"
                got.append(h[:s].view(d) if a else None)
            res.append(got)
        return res

    def assert_ranges(self, before, ref_inv, what):
        """Every rank's own GPU range is ref_inv's; without `before`, that is all; with it, every GPU outside the range is
        as the rank held it in `before`."""
        for r, inv in enumerate(self.inventories()):
            g0, g1 = self.gpu_range(r)
            assert inv[g0:g1].tobytes() == ref_inv[g0:g1].tobytes(), f"{what}: rank {r} own range differs from the oracle"
            if before is not None:
                assert inv[:g0].tobytes() == before[r][:g0].tobytes() and inv[g1:].tobytes() == before[r][g1:].tobytes(), \
                    f"{what}: rank {r} wrote GPUs outside its range"

    def assert_synced(self, state, what):
        """After an inventory sync every rank holds `state` whole (world 1: no sync is needed)."""
        if self.world > 1:
            self.sync_inventory()
        for r, inv in enumerate(self.inventories()):
            assert inv.tobytes() == state.tobytes(), f"{what}: rank {r} inventory after the sync differs from the oracle"


def _raw(outs):
    """The host copy of every rank's whole output buffers, for a failed call's checks."""
    return [[t.cpu().numpy() for t in o] for o in outs]


def unsuitable(W, claims, pod_off, cands=None, flags=0, n_pair=None, sentinel=0x5C, expect=0):
    """dra_unsuitable_batch_global_device: every rank's bitmap, no bit set past n_pair."""
    cn, co = (None, None) if cands is None else cands
    n_pod = len(pod_off) - 1
    if n_pair is None:
        n_pair = n_pod * W.n_node if co is None else int(co[-1])
    keep = [dev(claims), dev(pod_off)] + ([None, None] if cn is None else [dev(cn), dev(co)])
    nb = (n_pair + 7) // 8
    outs = W.outputs([nb], sentinel)
    W.each(lambda r, c: c.unsuitable_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), n_pod, ptr(keep[2]),
                                                   ptr(keep[3]), n_pair, outs[r][0].data_ptr(), flags), expect)
    if expect:
        return _raw(outs)
    bits = [got[0] for got in W.read(outs, [nb], [np.uint8], ["the bitmap"], [True], sentinel)]
    for r, b in enumerate(bits):
        assert n_pair % 8 == 0 or b[-1] >> (n_pair % 8) == 0, f"rank {r}: bits past n_pair are set"
    return bits


def allocate(W, claims, out_off, n_out, flags=0):
    """The sharded claim Allocate (dra_allocate_batch_global_device): every rank's gathered table."""
    keep = [dev(claims), None if out_off is None else dev(out_off)]
    W.each(lambda r, c: c.allocate_global_device(keep[0].data_ptr(), len(claims), ptr(keep[1]), n_out, flags))
    return [c.gather_read(np.zeros(n_out, dtype=W.pkg.records.OUT_DTYPE)) for c in W.ctxs]


def pods(W, claims, pod_off, out_off, n_out, flags=0, expect=0):
    """dra_allocate_pods_batch_global_device: every rank's gathered table."""
    keep = [dev(claims), dev(pod_off), None if out_off is None else dev(out_off)]
    W.each(lambda r, c: c.allocate_pods_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), len(pod_off) - 1,
                                                      ptr(keep[2]), n_out, flags), expect)
    if expect:
        return None
    return [c.gather_read(np.zeros(n_out, dtype=W.pkg.records.OUT_DTYPE)) for c in W.ctxs]


def place(W, claims, pod_off, cands, out_off, n_out, flags=0, n_pair=None, sentinel=0x5C, expect=0):
    """dra_place_pods_batch_global_device: every rank's (gathered table, pod_node)."""
    cn, co = (None, None) if cands is None else cands
    n_pod = len(pod_off) - 1
    if n_pair is None:
        n_pair = 0 if co is None else int(co[-1])
    keep = [dev(claims), dev(pod_off), None if out_off is None else dev(out_off)] + \
        ([None, None] if co is None else [dev(cn), dev(co)])
    outs = W.outputs([n_pod * 4], sentinel)
    W.each(lambda r, c: c.place_pods_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), n_pod, ptr(keep[3]),
                                                   ptr(keep[4]), n_pair, ptr(keep[2]), n_out, outs[r][0].data_ptr(), flags),
           expect)
    if expect:
        return _raw(outs)
    nodes = W.read(outs, [n_pod * 4], [np.uint32], ["pod_node"], [True], sentinel)
    return [(c.gather_read(np.zeros(n_out, dtype=W.pkg.records.OUT_DTYPE)), nd[0]) for c, nd in zip(W.ctxs, nodes)]


PREEMPT_NAMES = ("pair_status", "pair_victims", "pod_node", "pod_status", "n_victims", "victims", "pair_violations",
                 "pod_violations")


def preempt(W, claims, pod_off, prio, run, cands=None, max_victims=16, flags=0, pairs=True, pdb=False, bud=None,
            sentinel=0x5C, expect=0, asked=None):
    """dra_preempt_batch_global_device, or with pdb=True dra_preempt_pdb_batch_global_device with the budgets `bud` (None:
    a null struct): every rank's six or eight outputs, the per-pair ones None unless `pairs`.  `run`: the running pods of
    every rank, or a list of one per rank.  asked: one flag per output in PREEMPT_NAMES order, False for an output passed
    as NULL (read back as None), instead of what `pairs` says."""
    n_pod = len(pod_off) - 1
    cn, co = (None, None) if cands is None else cands
    n_pair = n_pod * W.n_node if co is None else int(co[-1])
    keep = [dev(claims), dev(pod_off), dev(prio)] + ([None, None] if cn is None else [dev(cn), dev(co)])
    sizes = [n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * max_victims * 4] + ([n_pair * 4, n_pod * 4] if pdb else [])
    if asked is None:
        asked = [pairs, pairs, True, True, True, True] + ([pairs, True] if pdb else [])
    assert len(asked) == len(sizes)
    outs = W.outputs(sizes, sentinel)

    def call(r, c):
        rs = (run[r] if isinstance(run, list) else run).struct
        p = [t.data_ptr() if a else None for t, a in zip(outs[r], asked)]
        victims = p[5] if max_victims else None
        if pdb:
            c.preempt_pdb_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                        ptr(keep[3]), ptr(keep[4]), n_pair, rs, None if bud is None else bud.struct,
                                        p[0], p[1], p[6], p[2], p[3], p[4], p[7], victims, max_victims, flags)
        else:
            c.preempt_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                    ptr(keep[3]), ptr(keep[4]), n_pair, rs, *p[:5], victims, max_victims, flags)

    W.each(call, expect)
    if expect:
        return _raw(outs)
    dt = [np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32, np.uint32, np.uint32]
    res = W.read(outs, sizes, dt, PREEMPT_NAMES, asked, sentinel)
    for got in res:
        got[5] = got[5].reshape(n_pod, max_victims)
    return res


CAPACITY_NAMES = ("pair_copies", "pair_stop", "pod_total", "pod_nodes")


def capacity(W, claims, pod_off, cands=None, max_copies=64, flags=0, want=(True, True, True), sentinel=0x5C, expect=0):
    """dra_pod_capacity_batch_global_device: every rank's four outputs, the optional ones None unless `want`."""
    n_pod = len(pod_off) - 1
    cn, co = (None, None) if cands is None else cands
    n_pair = n_pod * W.n_node if co is None else int(co[-1])
    keep = [dev(claims), dev(pod_off)] + ([None, None] if cn is None else [dev(cn), dev(co)])
    sizes = [n_pair * 2, n_pair, n_pod * 8, n_pod * 4]
    asked = [True] + list(want)
    outs = W.outputs(sizes, sentinel)
    W.each(lambda r, c: c.pod_capacity_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), n_pod, ptr(keep[2]),
                                                     ptr(keep[3]), n_pair, max_copies,
                                                     *[t.data_ptr() if a else None for t, a in zip(outs[r], asked)],
                                                     flags=flags), expect)
    if expect:
        return _raw(outs)
    return W.read(outs, sizes, [np.uint16, np.uint8, np.uint64, np.uint32], CAPACITY_NAMES, asked, sentinel)


def preempt_place(W, claims, pod_off, prio, run, cands, out_off, n_out, flags=0, sentinel=0x5C, expect=0):
    """dra_preempt_place_batch_global_device: every rank's (table, pod_node, pod_status, evicted_by).  A call without
    pending pods writes no table: its table is then zeros."""
    R = W.pkg.records
    n_pod, n_run = len(pod_off) - 1, run.struct.n_pod
    cn, co = (None, None) if cands is None else cands
    keep = [dev(claims), dev(pod_off), dev(prio), None if out_off is None else dev(out_off)] + \
        ([None, None] if cn is None else [dev(cn), dev(co)])
    sizes = [n_pod * 4, n_pod, n_run * 4]
    outs = W.outputs(sizes, sentinel)
    W.each(lambda r, c: c.preempt_place_global_device(keep[0].data_ptr(), len(claims), keep[1].data_ptr(), keep[2].data_ptr(),
                                                      n_pod, ptr(keep[4]), ptr(keep[5]), 0 if co is None else int(co[-1]),
                                                      run.struct, ptr(keep[3]), n_out, *[t.data_ptr() for t in outs[r]],
                                                      flags), expect)
    if expect:
        return _raw(outs)
    res = W.read(outs, sizes, [np.uint32, np.uint8, np.uint32], ("pod_node", "pod_status", "evicted_by"), [True] * 3,
                 sentinel)
    return [(c.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE)) if n_out and n_pod else np.zeros(n_out, R.OUT_DTYPE), *got)
            for c, got in zip(W.ctxs, res)]


def deallocate(W, claims, out_off, n_out, state=None, what="", out=None, ptrs=None, expect=0):
    """dra_deallocate_batch_global_device: `out` is one OutRec array uploaded for all ranks, or `ptrs` one device pointer
    per rank (each rank's gathered table).  A call that succeeds enqueues exactly two kernels on every rank; with `state`,
    the oracle's state after the call, every rank's own range is checked against it and nothing outside it may change."""
    keep = [dev(claims), None if out_off is None else dev(out_off)]
    if ptrs is None:
        keep.append(dev(out))
        ptrs = [keep[2].data_ptr()] * W.world
    before, l0 = W.inventories(), [c.launch_count() for c in W.ctxs]
    W.each(lambda r, c: c.deallocate_global_device(keep[0].data_ptr(), len(claims), ptr(keep[1]), ptrs[r], n_out), expect)
    if expect:
        return
    assert [c.launch_count() - l for c, l in zip(W.ctxs, l0)] == [2] * W.world, f"{what}: launches"
    if state is not None:
        W.assert_ranges(before, state, what)


# ---- a world-1 context on a sub-range shard [lo, hi): the kept claims' slots and the shard's GPUs against the oracle ----
def kept(w, lo, hi, stray):
    node = w.claims["node"].astype(np.int64)
    return np.where(node >= w.n_node, bool(stray), (node >= lo) & (node < hi))


def _slots_of(pkg, w, keep):
    """OutRec slots of the claims in `keep` (bool mask over the claims)."""
    sl = pkg.records.claim_slots(w.claims, w.n_node).astype(np.int64)
    start = (np.arange(w.n_claim) if w.out_off is None else w.out_off.astype(np.int64))[keep]
    n = sl[keep]
    first = np.repeat(np.cumsum(n) - n, n)
    m = np.zeros(w.n_out, dtype=bool)
    m[np.repeat(start, n) + np.arange(int(n.sum())) - first] = True
    return m


def shard_call(pkg, c, w, d_claims, d_off, lo, hi, stray, ref, ref_inv, what):
    """One sharded call on [lo, hi): kept slots and the shard's inventory slice against the oracle, the rest untouched."""
    R = pkg.records
    c.allocate_global_device(d_claims.data_ptr(), w.n_claim, None if d_off is None else d_off.data_ptr(), w.n_out,
                             pkg.api.F_FRESH_INVENTORY)
    got = c.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE))
    keep = kept(w, lo, hi, stray)
    assert 0 < keep.sum() < w.n_claim, f"{what}: the shard must keep some claims and drop others"
    m = _slots_of(pkg, w, keep)
    if got[m].tobytes() != ref[m].tobytes():
        bad = np.nonzero(got.view(np.uint64)[m] != ref.view(np.uint64)[m])[0]
        raise AssertionError(f"{what}: {len(bad)} kept OutRecs differ, first at slot {np.nonzero(m)[0][bad[0]]}")
    inv = c.get_inventory()
    g0, g1 = int(w.node_off[lo]), int(w.node_off[hi])
    assert inv[g0:g1].tobytes() == ref_inv[g0:g1].tobytes(), f"{what}: shard inventory differs"
    return got, m, c.last_chain()
