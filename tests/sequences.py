"""Long seeded sequences of library calls over one inventory, and the model that replays them on the CPU oracle.

A long-lived driver process makes thousands of calls on one context: Allocate batches of changing size and content, with
and without DRA_F_FRESH_INVENTORY and out_off, Deallocate of earlier batches, UnsuitableNodes, pods Allocate, place pods,
preemption with and without disruption budgets, preempt and place, pod capacity, and now and then a new inventory,
selector table or placement table.  The preemption calls take as running pods the records the sequence itself placed and
still holds, and preempt and place evicts some of them: a later Deallocate of their batch releases only what is left.
`make_sequence` draws such a sequence from a seed; `Model` applies it to oracle/oracle.py and the pod-call oracles and
records, for every step, the output the library must return and the state it must be left in.  Used by
tests/test_sequence_model.py (the model against oracle/naive.py and the naive pod-call restatements) and
tests/test_gpu_sequences.py (every context path against the model)."""
from __future__ import annotations

import importlib
from dataclasses import dataclass, field

import numpy as np

import capacity_oracle
import place_oracle
import pod_oracles
import preempt_oracle
import preempt_place_oracle

R = importlib.import_module("k8s-dra-driver_b200").records
synth = importlib.import_module("k8s-dra-driver_b200").synth

STAGED_CAP = 11_117          # most claims whose staged layout fits the single-launch kernel (the resident capacity)
PIECE = 256                  # claims per staged piece of the single-launch kernel
F_NODE_SORTED, F_FRESH, F_EXHAUSTIVE = 0x1, 0x2, 0x4
NONE = 0xFFFFFFFF
SENTINEL = np.frombuffer(bytes([0xA5, 0x5A, 0xC3, 0x3C, 0x96, 0x69, 0xE1, 0x1E]), dtype=R.OUT_DTYPE)[0]
RUN_PRIO = 100               # a held pod's priority is drawn from [0, RUN_PRIO); a pending pod's from [-1, RUN_PRIO + 20)
EVICTED = R.ST_POD           # the status an evicted pod's slots are held with: not OK, so never released again
PREEMPT_KINDS = ("preempt", "preempt_pdb", "preempt_place")
POD_CALLS = ("place",) + PREEMPT_KINDS + ("capacity",)
KINDS = {"alloc", "error", "sorted", "sorted_bad", "dealloc", "unsuitable", "pods", "selectors", "table", "reset",
         "set_inventory", "calibrate", "idle", "restart"} | set(POD_CALLS) | {k + "_bad" for k in POD_CALLS}


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
    #                               reset | set_inventory | calibrate | idle | restart | place | capacity | preempt |
    #                               preempt_pdb | preempt_place, and each of the last five + "_bad": a call it refuses
    claims: np.ndarray | None = None
    out_off: np.ndarray | None = None
    n_out: int = 0
    flags: int = 0
    pod_off: np.ndarray | None = None
    cand_nodes: np.ndarray | None = None
    cand_off: np.ndarray | None = None
    batches: list = field(default_factory=list)      # dealloc: indices of the earlier steps whose records are released;
    #                                                  preemption: of the held batches the running pods come from (Model)
    arg: object = None            # selectors: on/off; table: index; set_inventory: "base" | "live"; capacity: max_copies;
    #                               preempt, preempt_pdb: max_victims
    prio: np.ndarray | None = None                   # per pod (per claim for Allocate batches): a pending pod's priority,
    #                                                  or the one a placed pod keeps while it runs
    pdb_allowed: np.ndarray | None = None            # preempt_pdb: each budget's disruptionsAllowed
    expect: object = None         # filled by Model: OutRecs, UnsuitableNodes bits, or the tuple of a pod call's outputs
    #                               (None: the call is refused)
    live_after: np.ndarray | None = None             # filled by Model

    @property
    def base(self):
        """the call a refused step makes"""
        return self.kind[:-4] if self.kind.endswith("_bad") and self.kind != "sorted_bad" else self.kind

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

    def held_prio(self, n):
        return self.rng.integers(0, RUN_PRIO, size=n).astype(np.int32)

    def pending_prio(self, n):
        """a fifth outrank no held pod (-1), the rest some or all of them"""
        p = self.rng.integers(0, RUN_PRIO + 20, size=n)
        return np.where(self.rng.random(n) < 0.2, -1, p).astype(np.int32)

    def pod_claims(self, n_pod, most):
        """n_pod pods of 1 .. most claims: (claims, pod_off)"""
        sizes = self.rng.integers(1, most + 1, size=n_pod)
        pod_off = np.zeros(n_pod + 1, dtype=np.uint32)
        pod_off[1:] = np.cumsum(sizes)
        return self.window(int(pod_off[-1])), pod_off

    def cands(self, n_pod):
        """(None, None), the dense form, or 0-5 candidates per pod, a few naming no node, some repeated"""
        rng, nn = self.rng, self.inv.n_node
        if rng.random() < 0.4:
            return None, None
        cand_off = np.zeros(n_pod + 1, dtype=np.uint32)
        cand_off[1:] = np.cumsum(rng.integers(0, 6, size=n_pod))
        cand = rng.integers(0, nn + 2, size=int(cand_off[-1])).astype(np.uint32)
        again = np.nonzero(rng.random(len(cand)) < 0.15)[0]
        again = again[again > 0]
        cand[again] = cand[again - 1]
        return cand, cand_off

    def alloc(self, n, with_off, flags, n_out=None):
        c = self.window(n)
        nn = self.inv.n_node
        if not with_off:
            c["count"] = np.where((c["kind"] == R.KIND_GPU) & (c["count"] > 1) & (c["count"] <= 32), 1, c["count"])
            return Step("alloc", c, None, n, flags, prio=self.held_prio(n))
        if n_out is not None and not set_slots(c, nn, n_out):
            n_out = None
        off, total = R.out_offsets(c, nn)
        return Step("alloc", c, off, total, flags, prio=self.held_prio(n))

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
        c, pod_off = self.pod_claims(n_pod, 5)
        c["node"] = np.repeat(c["node"][pod_off[:-1]], np.diff(pod_off))
        off, total = R.out_offsets(c, nn)
        return Step("pods", c, off, total, F_EXHAUSTIVE if rng.random() < 0.5 else 0, pod_off=pod_off,
                    prio=self.held_prio(n_pod))

    def placed(self, kind, n_pod, flags, prio):
        """place / preempt_place: pods of 1-5 claims whose node fields are left as drawn (the calls ignore them), slots
        counted as if every claim named a node (§13)"""
        c, pod_off = self.pod_claims(n_pod, 5)
        at = c.copy()
        at["node"] = 0
        off, total = R.out_offsets(at, self.inv.n_node)
        cn, co = self.cands(n_pod)
        return Step(kind, c, off, total, flags, pod_off=pod_off, cand_nodes=cn, cand_off=co, prio=prio)

    def place(self):
        n_pod = int(self.rng.integers(1, 61))
        return self.placed("place", n_pod, int(self.rng.choice([0, F_EXHAUSTIVE, F_FRESH])), self.held_prio(n_pod))

    def preempt(self, kind):
        rng = self.rng
        n_pod = int(rng.integers(1, 41))
        flags = F_EXHAUSTIVE if rng.random() < 0.5 else 0
        if kind == "preempt_place":
            return self.placed(kind, n_pod, flags, self.pending_prio(n_pod))
        c, pod_off = self.pod_claims(n_pod, 4)
        cn, co = self.cands(n_pod)
        s = Step(kind, c, None, 0, flags, pod_off=pod_off, cand_nodes=cn, cand_off=co, arg=int(rng.choice([0, 3, 64])),
                 prio=self.pending_prio(n_pod))
        if kind == "preempt_pdb":
            s.pdb_allowed = rng.choice([0, 1, 2, 1 << 30], size=int(rng.integers(1, 5)),
                                       p=[0.55, 0.15, 0.15, 0.15]).astype(np.int32)
        return s

    def capacity(self):
        s = self.unsuitable()
        s.kind, s.arg = "capacity", int(self.rng.choice([1, 5, 64, 300]))
        return s

    def refused(self, kind):
        """One call of `kind` that the library refuses: a cand_off that is not monotone (place, capacity), a running
        pod whose OK slots lie on two nodes (preempt, preempt_pdb: added by the Model, see `two_node_pod`), or
        DRA_F_FRESH_INVENTORY given to preempt and place."""
        while True:
            s = {"place": self.place, "capacity": self.capacity}.get(kind, lambda: self.preempt(kind))()
            if kind in ("place", "capacity") and (s.cand_off is None or len(s.cand_off) < 3 or s.cand_off[-1] == 0):
                continue
            break
        if kind in ("place", "capacity"):
            s.cand_off = s.cand_off.copy()
            s.cand_off[1] = s.cand_off[-1] + 1
        elif kind == "preempt_place":
            s.flags |= F_FRESH
        s.kind += "_bad"
        return s

    def unsuitable(self):
        rng, nn = self.rng, self.inv.n_node
        n_pod = int(rng.integers(1, 40))
        c, pod_off = self.pod_claims(n_pod, 4)
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
        return Step("sorted_bad" if bad else "sorted", c, None, len(c), F_NODE_SORTED, prio=self.held_prio(len(c)))

    def error(self):
        s = self.alloc(int(self.rng.integers(8, 2000)), True, 0)
        s.kind = "error"
        s.out_off = s.out_off.copy()
        s.out_off[int(self.rng.integers(0, len(s.out_off)))] = s.n_out + int(self.rng.integers(0, 3))
        return s


def make_sequence(inv: Inventory, n_steps: int, seed: int, *, max_claims: int = 2 * STAGED_CAP,
                  selectors: bool = True, calibrate: bool = True) -> list:
    """n_steps (about) seeded steps over `inv`.  Every step kind appears; the error batch, the calibration, the idle wait,
    the restart and one refused call of each pod call appear once each, at fixed fractions of the sequence, and so do one
    refused node-sorted batch and one set_inventory of the live state besides the drawn ones."""
    g = _Gen(inv, seed, max_claims, selectors)
    rng = g.rng
    steps = []
    # set_inventory is also drawn, but too rarely for every sequence to have one; the one here comes late, so the
    # preemption steps before it see running sets grown over most of the sequence (it clears the held records)
    once = [(0.15, "sorted_bad"), (0.25, "place_bad"), (0.3, "error"), (0.4, "capacity_bad"), (0.55, "idle"),
            (0.6, "preempt_bad"), (0.7, "restart"), (0.75, "preempt_pdb_bad"), (0.8, "set_inventory"),
            (0.9, "preempt_place_bad")]
    cap = min(STAGED_CAP, max_claims)                    # runs at the staged capacity, one past it, and 2 x it in OutRecs
    runs = {int(n_steps * 0.1): (cap, False, None), int(n_steps * 0.2): (cap + 1, False, None),
            int(n_steps * 0.35): (cap // 2, True, 2 * cap), int(n_steps * 0.5): (cap, True, 2 * cap + 1),
            int(n_steps * 0.65): (cap, True, None), int(n_steps * 0.85): (1, True, None)}
    if calibrate:
        once.append((0.45, "calibrate"))
    once = sorted((int(n_steps * f), s) for f, s in once)
    live = []                                            # steps whose records are still allocated
    turn = 0
    while len(steps) < n_steps:
        special = [s for k, s in once if k <= len(steps)]
        once = once[len(special):]
        new = []
        for s in special:
            if s == "error":
                new += [g.error(), Step("reset")]
            elif s == "sorted_bad":
                new.append(g.sorted_batch(bad=True))
            elif s.endswith("_bad"):
                new.append(g.refused(s[:-4]))
            elif s == "set_inventory":
                new.append(Step(s, arg="live"))
            else:
                new.append(Step(s))
        for k in [k for k in sorted(runs) if k <= len(steps)]:
            new += g.alloc_run(*runs.pop(k))
        if not new:
            r = rng.random()
            if r < 0.4:
                new = g.alloc_run()
            elif r < 0.49 and live:
                pick = sorted(rng.choice(len(live), size=int(rng.integers(1, min(4, len(live)) + 1)), replace=False))
                new = [Step("dealloc", batches=[live[i] for i in pick])]
            elif r < 0.58:
                new = [g.unsuitable()]
            elif r < 0.635:
                new = [g.pods()]
            elif r < 0.9:                                # the pod calls in turn, so each has its share of the steps
                kind = POD_CALLS[turn % len(POD_CALLS)]
                turn += 1
                new = [g.place() if kind == "place" else g.capacity() if kind == "capacity" else g.preempt(kind)]
            elif r < 0.935:
                new = [g.sorted_batch(bad=rng.random() < 0.15)]
            elif r < 0.955 and selectors:
                g.sel_on = not g.sel_on
                new = [Step("selectors", arg=g.sel_on)]
            elif r < 0.965:
                new = [Step("table", arg=int(rng.integers(0, 2)))]
            elif r < 0.98:
                new = [Step("reset")]
            else:
                new = [Step("set_inventory", arg="live" if rng.random() < 0.6 else "base")]
        for s in new:
            i = len(steps)
            steps.append(s)
            if s.kind == "dealloc":
                live = [b for b in live if b not in s.batches]
            elif s.kind in ("alloc", "sorted", "pods", "place", "preempt_place"):
                if s.kind in ("alloc", "place") and s.flags & F_FRESH:
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


@dataclass
class Held:
    """The records of one batch still allocated, as Deallocate takes them, split into the units that run as one pod
    each: a pod of a pods, place or preempt_place step, a claim of an Allocate batch."""
    claims: np.ndarray            # a placed pod's claims name its node (§13 and §15 never write the node field)
    out_off: np.ndarray | None
    out: np.ndarray               # a copy of the call's output; an evicted unit's slots are EVICTED
    unit_off: np.ndarray          # unit u = claims unit_off[u] .. unit_off[u + 1]
    prio: np.ndarray              # per unit
    table: int                    # the placement table the batch was placed under
    gone: np.ndarray              # per unit: evicted, so no longer running

    def evict(self, units, n_node):
        """Units released by preempt and place: their OK slots become EVICTED, and they stop running."""
        have_off = self.out_off is not None
        base = self.out_off.astype(np.int64) if have_off else np.arange(len(self.claims))
        n = R.claim_slots(self.claims, n_node, have_off)
        for u in units:
            for i in range(int(self.unit_off[u]), int(self.unit_off[u + 1])):
                st = self.out["status"][base[i]: base[i] + n[i]]
                st[st == R.ST_OK] = EVICTED
            self.gone[u] = True


def held(s, out, pod_node, table, node_off):
    """The Held record of step s, whose call wrote `out` (and `pod_node`, for place and preempt_place).  Asserts the two
    rules the running pods rest on: a placed pod is held with its claims naming its node, which holds every OK slot of
    the pod (an unplaced pod has none), and every claim has the same slots when counted with an out_off (as the running
    pods are) as in the call that placed it."""
    n_node = len(node_off) - 1
    claims = s.claims
    unit_off = np.arange(len(claims) + 1, dtype=np.uint32) if s.pod_off is None else s.pod_off
    if pod_node is not None:
        claims = claims.copy()
        claims["node"] = np.repeat(np.where(pod_node == NONE, 0, pod_node), np.diff(unit_off))
        base = s.out_off if s.out_off is not None else np.arange(len(claims))
        sl = R.claim_slots(claims, n_node, s.out_off is not None)
        for p in range(len(pod_node)):
            for i in range(int(unit_off[p]), int(unit_off[p + 1])):
                ok = out[int(base[i]): int(base[i]) + int(sl[i])]
                gpu = ok["gpu"][ok["status"] == R.ST_OK].astype(np.int64)
                assert (pod_node[p] != NONE or not len(gpu)) and \
                    (np.searchsorted(node_off, gpu, side="right") - 1 == claims["node"][i]).all(), \
                    f"pod {p}: an OK slot off its node {pod_node[p]}"
    assert (R.claim_slots(claims, n_node, True) == R.claim_slots(claims, n_node, s.out_off is not None)).all(), \
        "a held claim's slots differ from the ones its batch wrote"
    return Held(claims, s.out_off, out.copy(), unit_off, s.prio, table, np.zeros(len(unit_off) - 1, dtype=bool))


@dataclass
class Running:
    """§14's running pods: every unit of the held batches not evicted, in placement order (the start order §14 breaks
    ties by); batch[r], unit[r]: where running pod r is held."""
    claims: np.ndarray
    pod_off: np.ndarray
    prio: np.ndarray
    out: np.ndarray
    out_off: np.ndarray
    batch: np.ndarray
    unit: np.ndarray

    def budgets(self, n_pdb):
        """run_pdb of a preempt_pdb step: a fifth of the pods under no budget, the others under budget prio % n_pdb"""
        return np.where(self.prio % 5 == 4, NONE, self.prio % n_pdb).astype(np.uint32)


def running(batches, helds) -> Running:
    cs, offs, outs, prios, sizes, bs, us, base = [], [], [], [], [], [], [], 0
    for b, h in zip(batches, helds):
        u = np.flatnonzero(~h.gone)
        lo, n = h.unit_off[u].astype(np.int64), np.diff(h.unit_off)[u].astype(np.int64)
        idx = np.repeat(lo - np.cumsum(n) + n, n) + np.arange(int(n.sum()))
        off = np.arange(len(h.claims)) if h.out_off is None else h.out_off.astype(np.int64)
        cs.append(h.claims[idx])
        offs.append(off[idx] + base)
        outs.append(h.out)
        prios.append(h.prio[u])
        sizes.append(n)
        bs.append(np.full(len(u), b))
        us.append(u)
        base += len(h.out)
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)        # noqa: E731
    pod_off = np.zeros(sum(len(x) for x in sizes) + 1, dtype=np.uint32)
    pod_off[1:] = np.cumsum(cat(sizes, np.int64))
    return Running(cat(cs, R.CLAIM_DTYPE), pod_off, cat(prios, np.int32), cat(outs, R.OUT_DTYPE), cat(offs, np.uint32),
                   cat(bs, np.int64), cat(us, np.int64))


def release(helds, run, evicted_by, n_node):
    """The running pods preempt and place evicted (evicted_by, one per pod of run): masked in their batches of
    helds (step index -> Held), and gone from every later running set."""
    r = np.flatnonzero(evicted_by != NONE)
    for b in np.unique(run.batch[r]):
        helds[int(b)].evict(run.unit[r][run.batch[r] == b], n_node)


def two_node_pod(run, gpus, node_off):
    """run with one more running pod, of two one-GPU claims whose OK slots lie on the first and the last GPU of the
    inventory, two different nodes: a fault §14 and §15 refuse.  (An inventory without GPUs on two nodes gets the other
    fault of that check instead: the last slot names a GPU past the inventory.)"""
    n_node, g = len(node_off) - 1, [0, len(gpus) - 1]
    node = np.searchsorted(node_off, g, side="right") - 1
    if len(gpus) == 0 or node[0] == node[1]:
        g, node = [0, len(gpus)], [0, 0]
    c = np.zeros(2, R.CLAIM_DTYPE)
    c["kind"], c["count"], c["node"] = R.KIND_GPU, 1, node
    assert (c["node"] < n_node).all()
    o = np.zeros(2, R.OUT_DTYPE)
    o["gpu"], o["profile"], o["status"] = g, R.PROFILE_GPU, R.ST_OK
    return Running(np.concatenate([run.claims, c]), np.append(run.pod_off, run.pod_off[-1] + 2).astype(np.uint32),
                   np.append(run.prio, 0).astype(np.int32), np.concatenate([run.out, o]),
                   np.append(run.out_off, [len(run.out), len(run.out) + 1]).astype(np.uint32),
                   np.append(run.batch, -1), np.append(run.unit, -1))


class Model:
    """The library's state as the oracle computes it: the live inventory, the pristine inventory last loaded, the records
    still allocated since the last FRESH batch, reset or set_inventory, the selector context and the placement table."""

    def __init__(self, inv: Inventory, oracle):
        self.inv, self.O = inv, oracle
        self.pristine = inv.gpus.copy()
        self.live = inv.gpus.copy()
        self.table = 0
        self.sel_on = False
        self.held = {}            # step index -> Held, in placement order

    def _sel(self):
        for set_selectors in (self.O.set_selectors, pod_oracles.set_selectors):     # (the pod oracles keep their own)
            if self.sel_on:
                set_selectors(self.inv.attrs, self.inv.sels)
            else:
                set_selectors()

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
            pod_oracles.set_selectors()
        return steps

    def keep(self, i, s, out, pod_node=None):
        self.held[i] = held(s, out, pod_node, self.table, self.inv.node_off)

    def step(self, i, s):
        O, inv = self.O, self.inv
        t = inv.tables[self.table]
        self._sel()
        if s.kind in ("alloc", "sorted"):
            src = self.pristine if s.flags & F_FRESH else self.live
            s.expect, self.live = O.allocate(src, inv.node_off, t, s.claims, s.out_off, s.n_out)
            if s.flags & F_FRESH:
                self.held = {}
            self.keep(i, s, s.expect)
        elif s.kind == "pods":
            s.expect, self.live = O.allocate_pods(self.live, inv.node_off, t, s.claims, s.pod_off, s.out_off, s.n_out, s.flags)
            self.keep(i, s, s.expect)
        elif s.kind == "dealloc":
            for b in s.batches:
                h = self.held.pop(b)
                self.live = O.deallocate(self.live, h.claims, h.out, h.out_off, inv.n_node)
        elif s.kind == "unsuitable":
            cn, co = s.cand_nodes, s.cand_off
            if cn is None:
                n_pod = len(s.pod_off) - 1
                cn = np.tile(np.arange(inv.n_node, dtype=np.uint32), n_pod)
                co = (np.arange(n_pod + 1, dtype=np.uint32) * inv.n_node).astype(np.uint32)
            s.expect = O.unsuitable(self.live, inv.node_off, t, s.claims, s.pod_off, cn, co, s.flags)
        elif s.base in POD_CALLS:
            try:
                self.pod_call(i, s, t)
            except ValueError:
                assert s.kind != s.base, f"step {i}: the oracle refuses a {s.kind} step"
                s.expect = None
                return
            assert s.kind == s.base, f"step {i}: the oracle accepts a {s.kind} step"
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

    def pod_call(self, i, s, t):
        """place, capacity and the preemption calls; raises ValueError where the oracle refuses the call"""
        inv, kind = self.inv, s.base
        exh = s.flags & F_EXHAUSTIVE
        common = (inv.node_off, t, s.claims, s.pod_off)
        if kind == "place":
            fresh = s.flags & F_FRESH
            out, node, live = place_oracle.place_pods(self.pristine if fresh else self.live, *common, s.cand_nodes,
                                                      s.cand_off, s.out_off, s.n_out, exh)
            s.expect, self.live = (out, node), live
            if fresh:
                self.held = {}
            self.keep(i, s, out, node)
            return
        if kind == "capacity":
            s.expect = capacity_oracle.capacity(self.live, *common, s.cand_nodes, s.cand_off, s.arg, exh)
            return
        s.batches = list(self.held)
        run = running(s.batches, [self.held[b] for b in s.batches])
        if s.kind in ("preempt_bad", "preempt_pdb_bad"):
            run = two_node_pod(run, self.live, inv.node_off)
        args = (self.live, *common, s.prio, run.claims, run.pod_off, run.prio, run.out)
        if kind == "preempt":
            s.expect = preempt_oracle.preempt(*args, run.out_off, s.cand_nodes, s.cand_off, s.arg, s.flags)
        elif kind == "preempt_pdb":
            s.expect = preempt_oracle.preempt_pdb(*args, run.budgets(len(s.pdb_allowed)), s.pdb_allowed, run.out_off,
                                                  s.cand_nodes, s.cand_off, s.arg, s.flags)
        else:
            res = preempt_place_oracle.preempt_place(*args, run.out_off, s.cand_nodes, s.cand_off, s.out_off, s.n_out,
                                                     s.flags)
            s.expect, self.live = res[:4], res[4]
            release(self.held, run, s.expect[3], inv.n_node)
            self.keep(i, s, s.expect[0], s.expect[1])

    # -- spec invariants of the state --------------------------------------------------------------------------------
    def check_invariants(self):
        inv, O = self.inv, self.O
        held = [(h.claims, h.out_off, h.out) for h in self.held.values()]
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
        for h in self.held.values():
            c, off, out, t = h.claims, h.out_off, h.out, inv.tables[h.table]
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
