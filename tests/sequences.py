"""Long seeded sequences of library calls over one inventory, and the model that replays them on the CPU oracle.

A long-lived driver process makes thousands of calls on one context: Allocate batches of changing size and content, with
and without DRA_F_FRESH_INVENTORY and out_off, Deallocate of earlier batches, UnsuitableNodes, pods Allocate, and now and
then a new inventory, selector table or placement table.  `make_sequence` draws such a sequence from a seed; `Model`
applies it to oracle/oracle.py and records, for every step, the output the library must return and the state it must be
left in.  Used by tests/test_sequence_model.py (the model against oracle/naive.py) and tests/test_gpu_sequences.py (every
context path against the model)."""
from __future__ import annotations

import importlib
from dataclasses import dataclass, field

import numpy as np

R = importlib.import_module("k8s-dra-driver_b200").records
synth = importlib.import_module("k8s-dra-driver_b200").synth

STAGED_CAP = 11_117          # most claims whose staged layout fits the single-launch kernel (the resident capacity)
PIECE = 256                  # claims per staged piece of the single-launch kernel
F_NODE_SORTED, F_FRESH, F_EXHAUSTIVE = 0x1, 0x2, 0x4
SENTINEL = np.frombuffer(bytes([0xA5, 0x5A, 0xC3, 0x3C, 0x96, 0x69, 0xE1, 0x1E]), dtype=R.OUT_DTYPE)[0]


@dataclass
class Inventory:
    """One inventory (node_off fixed for the whole sequence), its placement tables and the claim pools steps draw from."""
    name: str
    gpus: np.ndarray
    node_off: np.ndarray
    tables: list                  # [table as loaded, the same with one changed row]
    pool: np.ndarray              # claims (synth.mixed over these nodes; a few name no node at all)
    pool_sel: np.ndarray          # the same claims carrying selector ids (synth.with_selectors)
    attrs: np.ndarray
    sels: np.ndarray

    @property
    def n_node(self):
        return len(self.node_off) - 1


def inventory(name, gpus, node_off, table, seed):
    n_node = len(node_off) - 1
    assert n_node >= 2
    pool = synth.mixed(3 * STAGED_CAP, n_node, seed, invalid=True).claims
    pool["node"] = np.where(np.arange(len(pool)) % 211 == 7, 0xFFFFFFFF, pool["node"]).astype(np.uint32)
    w = synth.Workload(name, gpus, node_off, table, pool.copy())
    attrs, sels = synth.with_selectors(w, seed)
    t2 = table.copy()
    row = t2[int(gpus["model"][0]) if len(gpus) else 0]
    for p in range(R.MAX_PROFILES):                 # drop the lowest start of every profile that has more than one
        m = int(row[p]["start_mask"])
        if m & (m - 1):
            row[p]["start_mask"] = m & (m - 1)
    return Inventory(name, gpus.copy(), node_off.copy(), [table.copy(), t2], pool, w.claims, attrs, sels)


@dataclass
class Step:
    kind: str                     # alloc | error | sorted | sorted_bad | dealloc | unsuitable | pods | selectors | table |
    #                               reset | set_inventory | calibrate | idle | restart
    claims: np.ndarray | None = None
    out_off: np.ndarray | None = None
    n_out: int = 0
    flags: int = 0
    pod_off: np.ndarray | None = None
    cand_nodes: np.ndarray | None = None
    cand_off: np.ndarray | None = None
    batches: list = field(default_factory=list)      # dealloc: indices of the earlier steps whose records are released
    arg: object = None            # selectors: on/off; table: index; set_inventory: "base" | "live"
    expect: np.ndarray | None = None                 # filled by Model: OutRecs or UnsuitableNodes bits
    live_after: np.ndarray | None = None             # filled by Model

    def key(self):
        """What a captured graph of the host Allocate call is keyed on, besides the (fixed) buffers and the epoch."""
        return (self.kind, len(self.claims), self.out_off is not None, self.n_out, self.flags) if self.kind == "alloc" else None


def set_slots(c, n_node, target):
    """Raise the counts of valid GPU claims (up to 32) until the batch has `target` OutRec slots; False if it cannot."""
    need = target - int(R.claim_slots(c, n_node).sum())
    if need < 0:
        return False
    for i in np.nonzero((c["kind"] == R.KIND_GPU) & (c["node"] < n_node) & (c["count"] >= 1) & (c["count"] <= 32))[0]:
        if need <= 0:
            break
        add = min(need, 32 - int(c["count"][i]))
        c["count"][i] += add
        need -= add
    return need == 0


class _Gen:
    def __init__(self, inv, seed, max_claims, selectors):
        self.inv, self.rng, self.max_claims, self.selectors = inv, np.random.default_rng(seed), max_claims, selectors
        self.sel_on = False

    def window(self, n):
        pool = self.inv.pool_sel if (self.selectors and self.rng.random() < 0.3) else self.inv.pool
        at = int(self.rng.integers(0, len(pool) - n + 1))
        return pool[at: at + n].copy()

    def size(self):
        cap, rng = STAGED_CAP, self.rng
        r = rng.random()
        if r < 0.12:
            n = 1
        elif r < 0.2:
            n = int(rng.choice([cap, cap + 1]))
        elif r < 0.45:
            n = int(rng.integers(1, 9)) * PIECE + int(rng.integers(1, PIECE))          # not a multiple of a piece
        elif r < 0.55:
            n = int(rng.integers(1, 5)) * PIECE
        else:
            n = int(rng.integers(2, 3000))
        return max(1, min(n, self.max_claims))

    def alloc(self, n, with_off, flags, n_out=None):
        c = self.window(n)
        nn = self.inv.n_node
        if not with_off:
            c["count"] = np.where((c["kind"] == R.KIND_GPU) & (c["count"] > 1) & (c["count"] <= 32), 1, c["count"])
            return Step("alloc", c, None, n, flags)
        if n_out is not None and not set_slots(c, nn, n_out):
            n_out = None
        off, total = R.out_offsets(c, nn)
        return Step("alloc", c, off, total, flags)

    def alloc_run(self, n=None, with_off=None, n_out=None):
        """1-5 Allocate batches in a row; runs of 3 or more share one shape and flags (a captured graph replays them),
        and a run may end with the same shape under the other FRESH setting.  n / with_off / n_out: a run of this shape."""
        rng = self.rng
        k = int(rng.choice([1, 2, 3, 4, 5], p=[0.25, 0.2, 0.3, 0.15, 0.1])) if n is None else int(rng.integers(3, 5))
        flags = F_FRESH if rng.random() < 0.35 else 0
        if with_off is None:
            with_off = rng.random() < 0.6
        if n is None:
            n = self.size()
        if k < 3:
            return [self.alloc(self.size(), rng.random() < 0.6, F_FRESH if rng.random() < 0.35 else 0) for _ in range(k)]
        steps = [self.alloc(n, with_off, flags, n_out)]
        target = steps[0].n_out if with_off else None
        for _ in range(k - 1):
            steps.append(self.alloc(n, with_off, flags, target))
        if rng.random() < 0.5:
            steps.append(self.alloc(n, with_off, flags ^ F_FRESH, target))
        return steps

    def pods(self):
        rng, nn = self.rng, self.inv.n_node
        n_pod = int(rng.integers(1, 200))
        sizes = rng.integers(1, 6, size=n_pod)
        c = self.window(int(sizes.sum()))
        pod_off = np.zeros(n_pod + 1, dtype=np.uint32)
        pod_off[1:] = np.cumsum(sizes)
        c["node"] = np.repeat(c["node"][pod_off[:-1]], sizes)
        off, total = R.out_offsets(c, nn)
        return Step("pods", c, off, total, F_EXHAUSTIVE if rng.random() < 0.5 else 0, pod_off=pod_off)

    def unsuitable(self):
        rng, nn = self.rng, self.inv.n_node
        n_pod = int(rng.integers(1, 40))
        sizes = rng.integers(1, 5, size=n_pod)
        c = self.window(int(sizes.sum()))
        pod_off = np.zeros(n_pod + 1, dtype=np.uint32)
        pod_off[1:] = np.cumsum(sizes)
        flags = F_EXHAUSTIVE if rng.random() < 0.5 else 0
        if rng.random() < 0.5:
            return Step("unsuitable", c, None, 0, flags, pod_off=pod_off)
        k = rng.integers(0, 6, size=n_pod)
        cand_off = np.zeros(n_pod + 1, dtype=np.uint32)
        cand_off[1:] = np.cumsum(k)
        cand = rng.integers(0, nn + 2, size=int(cand_off[-1])).astype(np.uint32)       # a few name no node
        return Step("unsuitable", c, None, 0, flags, pod_off=pod_off, cand_nodes=cand, cand_off=cand_off)

    def sorted_batch(self, bad):
        c = self.window(max(2, self.size()))
        c["count"] = np.where((c["kind"] == R.KIND_GPU) & (c["count"] > 1) & (c["count"] <= 32), 1, c["count"])
        c = c[np.argsort(c["node"], kind="stable")]
        if bad:                                          # sorted but for one claim near the end that names node 0
            c["node"][len(c) - 1 - len(c) // 7] = 0
            c["node"][0] = max(int(c["node"][0]), 1)
        return Step("sorted_bad" if bad else "sorted", c, None, len(c), F_NODE_SORTED)

    def error(self):
        s = self.alloc(int(self.rng.integers(8, 2000)), True, 0)
        s.kind = "error"
        s.out_off = s.out_off.copy()
        s.out_off[int(self.rng.integers(0, len(s.out_off)))] = s.n_out + int(self.rng.integers(0, 3))
        return s


def make_sequence(inv: Inventory, n_steps: int, seed: int, *, max_claims: int = 2 * STAGED_CAP,
                  selectors: bool = True, calibrate: bool = True) -> list:
    """n_steps (about) seeded steps over `inv`.  Every step kind appears; the error batch, the calibration, the idle wait
    and the restart appear once each, at fixed fractions of the sequence."""
    g = _Gen(inv, seed, max_claims, selectors)
    rng = g.rng
    steps = []
    once = {int(n_steps * 0.3): "error", int(n_steps * 0.55): "idle", int(n_steps * 0.7): "restart"}
    cap = min(STAGED_CAP, max_claims)                    # runs at the staged capacity, one past it, and 2 x it in OutRecs
    runs = {int(n_steps * 0.1): (cap, False, None), int(n_steps * 0.2): (cap + 1, False, None),
            int(n_steps * 0.35): (cap // 2, True, 2 * cap), int(n_steps * 0.5): (cap, True, 2 * cap + 1),
            int(n_steps * 0.65): (cap, True, None), int(n_steps * 0.85): (1, True, None)}
    if calibrate:
        once[int(n_steps * 0.45)] = "calibrate"
    live = []                                            # steps whose records are still allocated
    while len(steps) < n_steps:
        special = [once.pop(k) for k in sorted(once) if k <= len(steps)]
        new = []
        for s in special:
            if s == "error":
                new += [g.error(), Step("reset")]
            else:
                new.append(Step(s))
        for k in [k for k in sorted(runs) if k <= len(steps)]:
            new += g.alloc_run(*runs.pop(k))
        if not new:
            r = rng.random()
            if r < 0.5:
                new = g.alloc_run()
            elif r < 0.62 and live:
                pick = sorted(rng.choice(len(live), size=int(rng.integers(1, min(4, len(live)) + 1)), replace=False))
                new = [Step("dealloc", batches=[live[i] for i in pick])]
            elif r < 0.72:
                new = [g.unsuitable()]
            elif r < 0.8:
                new = [g.pods()]
            elif r < 0.85:
                new = [g.sorted_batch(bad=rng.random() < 0.15)]
            elif r < 0.89 and selectors:
                g.sel_on = not g.sel_on
                new = [Step("selectors", arg=g.sel_on)]
            elif r < 0.92:
                new = [Step("table", arg=int(rng.integers(0, 2)))]
            elif r < 0.96:
                new = [Step("reset")]
            else:
                new = [Step("set_inventory", arg="live" if rng.random() < 0.6 else "base")]
        for s in new:
            i = len(steps)
            steps.append(s)
            if s.kind == "dealloc":
                live = [b for b in live if b not in s.batches]
            elif s.kind in ("alloc", "sorted", "pods"):
                if s.kind == "alloc" and s.flags & F_FRESH:
                    live = []
                live.append(i)
            elif s.kind in ("error", "reset", "set_inventory"):
                live = []
    return steps


def concat(batches):
    """One Deallocate call's (claims, out_off, out) for several batches."""
    cs, offs, outs, base = [], [], [], 0
    for c, off, out in batches:
        cs.append(c)
        offs.append((np.arange(len(c), dtype=np.uint32) if off is None else off.astype(np.uint32)) + np.uint32(base))
        outs.append(out)
        base += len(out)
    return np.concatenate(cs), np.concatenate(offs).astype(np.uint32), np.concatenate(outs)


class Model:
    """The library's state as the oracle computes it: the live inventory, the pristine inventory last loaded, the records
    still allocated since the last FRESH batch, reset or set_inventory, the selector context and the placement table."""

    def __init__(self, inv: Inventory, oracle):
        self.inv, self.O = inv, oracle
        self.pristine = inv.gpus.copy()
        self.live = inv.gpus.copy()
        self.table = 0
        self.sel_on = False
        self.held = {}            # step index -> (claims, out_off, out, table index)

    def _sel(self):
        if self.sel_on:
            self.O.set_selectors(self.inv.attrs, self.inv.sels)
        else:
            self.O.set_selectors()

    def run(self, steps, check=None):
        """Fills every step's expect / live_after; check(model, step) is called after each step."""
        try:
            for i, s in enumerate(steps):
                self.step(i, s)
                s.live_after = self.live.copy()
                if check:
                    check(self, s)
        finally:
            self.O.set_selectors()
        return steps

    def step(self, i, s):
        O, inv = self.O, self.inv
        t = inv.tables[self.table]
        self._sel()
        if s.kind in ("alloc", "sorted"):
            src = self.pristine if s.flags & F_FRESH else self.live
            s.expect, self.live = O.allocate(src, inv.node_off, t, s.claims, s.out_off, s.n_out)
            if s.flags & F_FRESH:
                self.held = {}
            self.held[i] = (s.claims, s.out_off, s.expect, self.table)
        elif s.kind == "pods":
            s.expect, self.live = O.allocate_pods(self.live, inv.node_off, t, s.claims, s.pod_off, s.out_off, s.n_out, s.flags)
            self.held[i] = (s.claims, s.out_off, s.expect, self.table)
        elif s.kind == "dealloc":
            for b in s.batches:
                c, off, out, _ = self.held.pop(b)
                self.live = O.deallocate(self.live, c, out, off, inv.n_node)
        elif s.kind == "unsuitable":
            cn, co = s.cand_nodes, s.cand_off
            if cn is None:
                n_pod = len(s.pod_off) - 1
                cn = np.tile(np.arange(inv.n_node, dtype=np.uint32), n_pod)
                co = (np.arange(n_pod + 1, dtype=np.uint32) * inv.n_node).astype(np.uint32)
            s.expect = O.unsuitable(self.live, inv.node_off, t, s.claims, s.pod_off, cn, co, s.flags)
        elif s.kind == "selectors":
            self.sel_on = bool(s.arg)
        elif s.kind == "table":
            self.table = int(s.arg)
        elif s.kind in ("error", "reset"):                # (the error batch is followed by a reset)
            self.live = self.pristine.copy()
            self.held = {}
        elif s.kind == "set_inventory":
            self.pristine = (self.live if s.arg == "live" else inv.gpus).copy()
            self.live = self.pristine.copy()
            self.held = {}
        else:
            assert s.kind in ("sorted_bad", "calibrate", "idle", "restart"), s.kind

    # -- spec invariants of the state --------------------------------------------------------------------------------
    def check_invariants(self):
        inv, O = self.inv, self.O
        held = [(c, off, out) for c, off, out, _ in self.held.values()]
        if held:
            c, off, out = concat(held)
            back = O.deallocate(self.live, c, out, off, inv.n_node)
        else:
            back = self.live
        assert back.tobytes() == self.pristine.tobytes(), "Deallocate of everything held does not restore the pristine state"
        share = self.pristine["share_cnt"].astype(np.int64).copy()
        mem = self.pristine["mem_free_mib"].astype(np.int64).copy()
        busy = self.pristine["busy"].astype(np.int64).copy()
        full = np.zeros(len(self.live), dtype=bool)
        for c, off, out, tix in self.held.values():
            t = inv.tables[tix]
            base = np.arange(len(c)) if off is None else off.astype(np.int64)
            sl = R.claim_slots(c, inv.n_node, off is not None).astype(np.int64)
            for i in np.nonzero(c["kind"] <= 2)[0]:
                for k in range(int(sl[i])):
                    o = out[base[i] + k]
                    if o["status"] != R.ST_OK:
                        continue
                    g = int(o["gpu"])
                    if c["kind"][i] == R.KIND_SHARED:
                        share[g] += 1
                        mem[g] -= int(c["mem_limit_mib"][i])
                    elif c["kind"][i] == R.KIND_GPU:
                        assert not full[g], "a GPU held twice"
                        full[g] = True
                    else:
                        e = t[int(self.live["model"][g]), int(o["profile"])]
                        assert int(o["size"]) == int(e["size"]) and (int(e["start_mask"]) >> int(o["start"])) & 1, \
                            "a MIG placement the table does not offer"
                        m = ((1 << int(o["size"])) - 1) << int(o["start"])
                        assert not busy[g] & m, "overlapping MIG placements"
                        busy[g] |= m
        assert (share <= 0xFFFF).all() and (share == self.live["share_cnt"]).all(), "share_cnt wrapped or drifted"
        assert (mem >= 0).all() and (mem == self.live["mem_free_mib"]).all()
        assert (busy == self.live["busy"]).all(), "busy holds more than the table placements of the held records"
        assert ((self.live["flags"] & R.GPU_FULL_ALLOCATED) != 0).tolist() == \
            ((self.pristine["flags"] & R.GPU_FULL_ALLOCATED != 0) | full).tolist()


def standard_inventories(n_sm: int):
    """The three inventories the GPU sequences run on: SMs - 1 nodes (the most the resident kernel serves), about 60 ragged
    nodes of 0-32 GPUs, and MIG nodes of up to 8 GPUs on a 16-slice table."""
    a = synth.mixed(10, n_sm - 1, 41)
    b = synth.mixed(10, 60, 42)
    h = synth.homog(10, 48, 43, max_width=8, wide16=True)
    return [inventory(f"mixed_{n_sm - 1}_nodes", a.gpus, a.node_off, a.table, 41),
            inventory("mixed_60_nodes", b.gpus, b.node_off, b.table, 42),
            inventory("mig16_48_nodes", h.gpus, h.node_off, h.table, 43)]
