"""CPU suite: the sequence model that tests/test_gpu_sequences.py compares every context path with.

The model (tests/sequences.py) carries the library's state across a long sequence of calls with the C oracle.  Here it is
replayed step by step by the pure-Python restatement (oracle/naive.py, plus Deallocate and UnsuitableNodes written from
spec §8/§9 below, and the naive restatements of place pods, preemption, preempt and place and pod capacity, with the
running pods, their evictions and what a later Deallocate releases restated here), and the spec's invariants of the state
are checked after every step."""
import copy

import numpy as np
import pytest

import capacity_oracle as CO
import place_oracle as PL
import preempt_oracle as PR
import preempt_place_oracle as PP
import sequences as S
from oracle import naive

NEW = S.POD_CALLS


def _dicts(a):
    return [{k: int(x[k]) for k in a.dtype.names} for x in a]


def _tuples(out):
    return [(int(o["gpu"]), int(o["start"]), int(o["size"]), int(o["profile"]), int(o["status"])) for o in out]


def _table(t):
    return [[(int(e["size"]), int(e["start_mask"])) for e in row] for row in t]


def _state(gpus):
    return [{k: g[k] for k in ("busy", "flags", "model", "mem_free_mib", "share_cnt")} for g in gpus]


class Naive:
    """The same sequence on oracle/naive.py: lists of dicts instead of records, no shared code with the C oracle."""

    def __init__(self, inv):
        self.inv = inv
        self.n_node = inv.n_node
        self.off = [int(x) for x in inv.node_off]
        self.base = _dicts(inv.gpus)
        self.pristine = copy.deepcopy(self.base)
        self.live = copy.deepcopy(self.base)
        self.table = 0
        self.held = {}

    def dealloc(self, claims, off, out):                     # spec §9
        have_off = off is not None
        for i, c in enumerate(claims):
            base = off[i] if have_off else i
            for k in range(naive._slots(c, self.n_node, have_off)):
                gpu, start, size, _, st = out[base + k]
                if st != 0:
                    continue
                g = self.live[gpu]
                if c["kind"] == 0:
                    g["flags"] &= ~2
                elif c["kind"] == 1:
                    g["busy"] &= ~(((1 << size) - 1) << start)
                else:
                    g["mem_free_mib"] += c["mem_limit_mib"]
                    g["share_cnt"] -= 1

    def unsuitable(self, claims, pod_off, cand_nodes, cand_off, exhaustive, t):      # spec §8 / §12
        bits = []
        for p in range(len(pod_off) - 1):
            pod = claims[pod_off[p]: pod_off[p + 1]]
            for n in cand_nodes[cand_off[p]: cand_off[p + 1]]:
                if n >= self.n_node:
                    bits.append(False)
                    continue
                moved = [dict(c, node=n) for c in pod]
                if exhaustive:
                    G = naive._state(self.live)
                    ok, _ = naive.eval_pod(G, self.off[n], self.off[n + 1], t, moved, self.n_node, True)
                else:
                    off, acc = [], 0
                    for c in moved:
                        off.append(acc)
                        acc += naive._slots(c, self.n_node, True)
                    out, _ = naive.allocate(self.live, self.off, t, moved, off)
                    ok = all(o[4] == 0 for o in out)
                bits.append(ok)
        return bits

    def keep(self, i, s, claims, off, out, pod_node=None):
        """held records of step i: one running pod per pod (per claim for Allocate batches), with its priority; a placed
        pod's claims name the node it was placed on (unplaced: node 0, it has no OK slot)"""
        units = [(k, k + 1) for k in range(len(claims))] if s.pod_off is None else \
            [(int(a), int(b)) for a, b in zip(s.pod_off[:-1], s.pod_off[1:])]
        if pod_node is not None:
            claims = [dict(c) for c in claims]
            for (a, b), n in zip(units, pod_node):
                for c in claims[a:b]:
                    c["node"] = 0 if n == S.NONE else n
        self.held[i] = dict(claims=claims, off=off, out=list(out), units=units, prio=[int(x) for x in s.prio],
                            gone=[False] * len(units))

    def running(self):
        """every held pod not evicted, in placement order: (claims, pod_off, prio, out, out_off, [(batch, unit)])"""
        rc, rpo, rpr, ro, roo, who = [], [0], [], [], [], []
        for b, h in self.held.items():
            for u, (a, z) in enumerate(h["units"]):
                if h["gone"][u]:
                    continue
                for k in range(a, z):
                    rc.append(h["claims"][k])
                    roo.append(len(ro) + (k if h["off"] is None else h["off"][k]))
                rpo.append(len(rc))
                rpr.append(h["prio"][u])
                who.append((b, u))
            ro += h["out"]
        return rc, rpo, rpr, ro, roo, who

    def evict(self, who, evicted_by):
        for r, p in enumerate(evicted_by):
            if p == S.NONE:
                continue
            b, u = who[r]
            h = self.held[b]
            h["gone"][u] = True
            for k in range(*h["units"][u]):
                base = k if h["off"] is None else h["off"][k]
                for j in range(base, base + naive._slots(h["claims"][k], self.n_node, h["off"] is not None)):
                    if h["out"][j][4] == 0:
                        h["out"][j] = h["out"][j][:4] + (S.EVICTED,)

    def _fresh(self, after, before):
        return [dict(g, node=g0["node"], rsvd=g0["rsvd"]) for g, g0 in zip(after, before)]

    def step(self, i, s):
        t = _table(self.inv.tables[self.table])
        claims = None if s.claims is None else _dicts(s.claims)
        off = None if s.out_off is None else [int(x) for x in s.out_off]
        pod_off = None if s.pod_off is None else [int(x) for x in s.pod_off]
        cands = None if s.cand_nodes is None else \
            [[int(x) for x in s.cand_nodes[a:b]] for a, b in zip(s.cand_off[:-1], s.cand_off[1:])]
        exh = bool(s.flags & S.F_EXHAUSTIVE)
        if s.kind in ("alloc", "sorted"):
            if s.flags & S.F_FRESH:
                self.live = copy.deepcopy(self.pristine)
                self.held = {}
            out, after = naive.allocate(self.live, self.off, t, claims, off)
            self.live = self._fresh(after, self.live)
            self.keep(i, s, claims, off, out)
            return out
        if s.kind == "pods":
            out, after = naive.allocate_pods(self.live, self.off, t, claims, pod_off, exh, off)
            self.live = self._fresh(after, self.live)
            self.keep(i, s, claims, off, out)
            return out
        if s.kind == "place":
            src = self.pristine if s.flags & S.F_FRESH else self.live
            out, node, after = PL.place_pods_naive(src, self.off, t, claims, pod_off, cands, exh, off)
            self.live = self._fresh(after, src)
            if s.flags & S.F_FRESH:
                self.held = {}
            self.keep(i, s, claims, off, out, node)
            return out, node
        if s.kind == "capacity":
            return CO.capacity_naive(self.live, self.off, t, claims, pod_off, cands, exh, s.arg)
        if s.kind in S.PREEMPT_KINDS:
            rc, rpo, rpr, ro, roo, who = self.running()
            prio = [int(x) for x in s.prio]
            if s.kind == "preempt":
                return PR.preempt_naive(self.live, self.off, t, claims, pod_off, prio, cands, exh, rc, rpo, rpr, ro, roo,
                                        s.arg)
            if s.kind == "preempt_pdb":
                pdb = [S.NONE if p % 5 == 4 else p % len(s.pdb_allowed) for p in rpr]
                return PR.preempt_naive_pdb(self.live, self.off, t, claims, pod_off, prio, cands, exh, rc, rpo, rpr, ro,
                                            pdb, [int(x) for x in s.pdb_allowed], roo, s.arg)
            out, node, status, evicted_by, after = PP.preempt_place_naive(self.live, self.off, t, claims, pod_off, prio,
                                                                          cands, exh, rc, rpo, rpr, ro, off, roo)
            self.live = self._fresh(after, self.live)
            self.evict(who, evicted_by)
            self.keep(i, s, claims, off, out, node)
            return out, node, status, evicted_by
        if s.kind == "dealloc":
            for b in s.batches:
                h = self.held.pop(b)
                self.dealloc(h["claims"], h["off"], h["out"])
        elif s.kind == "unsuitable":
            if s.cand_nodes is None:
                n_pod = len(pod_off) - 1
                cn, co = list(range(self.n_node)) * n_pod, [p * self.n_node for p in range(n_pod + 1)]
            else:
                cn, co = [int(x) for x in s.cand_nodes], [int(x) for x in s.cand_off]
            return self.unsuitable(claims, pod_off, cn, co, exh, t)
        elif s.kind == "table":
            self.table = int(s.arg)
        elif s.kind in ("error", "reset"):
            self.live = copy.deepcopy(self.pristine)
            self.held = {}
        elif s.kind == "set_inventory":
            self.pristine = copy.deepcopy(self.live if s.arg == "live" else self.base)
            self.live = copy.deepcopy(self.pristine)
            self.held = {}
        return None


def _small(n_node, seed):
    w = S.synth.mixed(10, n_node, seed)
    return S.inventory(f"small{n_node}", w.gpus, w.node_off, w.table, seed)


def _replay(oracle, inv, steps):
    """The model's outputs and states against the naive replay, step by step."""
    S.Model(inv, oracle).run(steps)
    nv = Naive(inv)
    for i, s in enumerate(steps):
        got = nv.step(i, s)
        if s.kind in ("alloc", "sorted", "pods"):
            assert _tuples(s.expect) == got, f"step {i} {s.kind}: OutRecs differ"
        elif s.kind in NEW:
            want = [_tuples(x) if x.dtype == S.R.OUT_DTYPE else x.tolist() for x in s.expect]
            assert want == [list(x) for x in got], f"step {i} {s.kind}: outputs differ"
        elif s.base in NEW:
            assert s.expect is None, f"step {i}: {s.kind} accepted"
        elif s.kind == "unsuitable":
            want = np.packbits(np.array(got, dtype=np.uint8), bitorder="little") if got else np.zeros(0, np.uint8)
            assert s.expect.tobytes() == want.tobytes(), f"step {i}: UnsuitableNodes bits differ"
        assert _state(_dicts(s.live_after)) == _state(nv.live), f"step {i} {s.kind}: state differs"


@pytest.mark.parametrize("n_node,seed", [(2, 1), (3, 2), (5, 3), (7, 4), (4, 5), (6, 6)])
def test_model_matches_naive_replay(oracle, n_node, seed):
    """About 30 steps on a small inventory: every output and every state of the model equals the naive replay."""
    inv = _small(n_node, seed)
    _replay(oracle, inv, S.make_sequence(inv, 30, seed, max_claims=24, selectors=False, calibrate=False))


@pytest.mark.parametrize("n_node,seed,n_steps,max_claims", [(3, 1, 200, 40), (5, 8, 200, 40), (6, 3, 200, 30),
                                                            (4, 4, 200, 40)])
def test_pod_calls_match_naive_replay(oracle, n_node, seed, n_steps, max_claims):
    """Longer sequences, so that every pod call runs several times on running sets built over many batches and preempt and
    place evicts some of their pods: the model's running pods, the masks of what was evicted and what a later Deallocate
    releases, against the naive replay's own."""
    inv = _small(n_node, seed)
    steps = S.make_sequence(inv, n_steps, seed, max_claims=max_claims, selectors=False, calibrate=False)
    _replay(oracle, inv, steps)
    kinds = [s.kind for s in steps]
    assert all(kinds.count(k) >= 3 for k in NEW), kinds
    assert any(s.kind == "preempt_place" and (s.expect[3] != S.NONE).any() for s in steps), "nothing evicted"


@pytest.mark.parametrize("n_node,seed,selectors", [(3, 11, False), (12, 12, True), (40, 13, True)])
def test_state_invariants_after_every_step(oracle, n_node, seed, selectors):
    """Deallocating every record still held restores the pristine state of the current epoch; share_cnt never wraps and
    counts exactly the SHARED records held; busy holds only table placements of the held records (spec §5, §7, §9)."""
    inv = _small(n_node, seed)
    steps = S.make_sequence(inv, 150, seed, max_claims=3000, selectors=selectors, calibrate=False)
    S.Model(inv, oracle).run(steps, check=lambda m, s: m.check_invariants())


def test_invariants_catch_a_lost_record(oracle):
    """The invariant check is sharp: a model that forgets one held batch no longer deallocates back to the pristine state."""
    inv = _small(5, 21)
    steps = S.make_sequence(inv, 40, 21, max_claims=200, calibrate=False)
    m = S.Model(inv, oracle)
    for i, s in enumerate(steps):
        m.step(i, s)
        live = [k for k, h in m.held.items() if (h.out["status"] == 0).any()]
        if live:
            del m.held[live[0]]
            with pytest.raises(AssertionError):
                m.check_invariants()
            return
    pytest.fail("no batch placed anything")


def _first_eviction(oracle):
    """The model run up to the first preempt and place step that evicts a held pod: (model, steps, the batches it
    evicted from)."""
    inv = _small(12, 12)
    steps = S.make_sequence(inv, 150, 12, max_claims=3000, calibrate=False)
    m = S.Model(inv, oracle)
    for i, s in enumerate(steps):
        m.step(i, s)
        hit = [b for b, h in m.held.items() if h.gone.any()]
        if hit:
            m.check_invariants()
            return m, steps, hit
    pytest.fail("no preempt and place step evicted anything")


def test_invariants_catch_an_unmasked_eviction(oracle):
    """The invariant check is sharp: a model that does not mask what preempt and place evicted still holds records the
    inventory no longer has."""
    m, steps, hit = _first_eviction(oracle)
    for b in hit:
        out = steps[b].expect if steps[b].kind in ("alloc", "sorted", "pods") else steps[b].expect[0]
        assert (m.held[b].out["status"] != out["status"]).any()
        m.held[b].out = out.copy()
    with pytest.raises(AssertionError):
        m.check_invariants()


def test_invariants_catch_an_eviction_released_again(oracle):
    """The invariant check is sharp: a model whose Deallocate of a batch releases the pods preempt and place evicted
    from it, again, leaves a state that Deallocate of everything still held does not restore."""
    m, steps, hit = _first_eviction(oracle)
    b = hit[0]
    h = m.held.pop(b)
    out = steps[b].expect if steps[b].kind in ("alloc", "sorted", "pods") else steps[b].expect[0]
    m.live = m.O.deallocate(m.live, h.claims, out, h.out_off, m.inv.n_node)
    with pytest.raises(AssertionError):
        m.check_invariants()


@pytest.mark.parametrize("n_node", [61, 132])
def test_sequence_covers_every_step_kind(oracle, n_node):
    """The GPU sequences' shape: every step kind (each pod call at least 8 times and refused once), the sizes at the staged
    capacity and twice it in OutRecs (each side of them), odd OutRec counts, sizes off the 256-claim piece, FRESH and
    out_off both ways, runs of three or more Allocate batches of one shape for a captured graph to replay, and Allocate
    batches in a row for the resident kernel."""
    w = S.synth.mixed(10, n_node, 40)
    inv = S.inventory("cover", w.gpus, w.node_off, w.table, 40)
    steps = S.make_sequence(inv, 400, 7)
    assert {s.kind for s in steps} == S.KINDS
    kinds = [s.kind for s in steps]
    assert all(kinds.count(k) >= 8 and kinds.count(k + "_bad") == 1 for k in NEW)
    assert any(s.kind == "place" and s.flags & S.F_FRESH for s in steps)
    # the pod calls' outcomes: evictions (of some pod an Allocate batch placed), EVICT and FITS, violated budgets, and
    # capacity counts ending both at max_copies and where the next copy does not fit
    evicted = set()
    S.Model(inv, oracle).run(steps, check=lambda m, s: evicted.update(steps[b].kind for b, h in m.held.items()
                                                                      if h.gone.any()))
    assert any((s.expect[3] != S.NONE).any() for s in steps if s.kind == "preempt_place") and "alloc" in evicted
    status = {int(x) for s in steps if s.kind == "preempt" for x in s.expect[3]}
    assert {PR.EVICT, PR.FITS} <= status, status
    assert any((s.expect[7] > 0).any() for s in steps if s.kind == "preempt_pdb")
    stops = {int(x) for s in steps if s.kind == "capacity" for x in s.expect[1]}
    assert {CO.ST_OK, CO.ST_POD} <= stops, stops
    al = [s for s in steps if s.kind == "alloc"]
    n = {len(s.claims) for s in al}
    outs = {s.n_out for s in al}
    cap = S.STAGED_CAP
    assert 1 in n and cap in n and cap + 1 in n, sorted(n)
    assert 2 * cap in outs and 2 * cap + 1 in outs
    assert any(x % 2 for x in outs) and any(x % S.PIECE for x in n)
    assert {(s.flags, s.out_off is not None) for s in al} == {(0, False), (0, True), (S.F_FRESH, False), (S.F_FRESH, True)}
    assert any(s.out_off is not None and (s.claims["count"] > 1).any() for s in al)
    keys = [s.key() for s in steps]
    runs = sum(1 for i in range(2, len(keys)) if keys[i] and keys[i] == keys[i - 1] == keys[i - 2])
    assert runs >= 10, runs
    switch = sum(1 for i in range(3, len(keys)) if keys[i] and keys[i - 1] and keys[i][:4] == keys[i - 1][:4] and
                 keys[i][4] != keys[i - 1][4] and keys[i - 1] == keys[i - 2] == keys[i - 3])
    assert switch >= 2, switch
    pairs = sum(1 for a, b in zip(steps, steps[1:]) if a.kind == b.kind == "alloc" and len(b.claims) <= cap)
    assert pairs >= 50, pairs
    assert [s.kind for s in steps].count("error") == 1 and steps[[s.kind for s in steps].index("error") + 1].kind == "reset"
    # the same seed gives the same sequence
    again = S.make_sequence(inv, 400, 7)
    assert all(a.kind == b.kind and (a.claims is None or a.claims.tobytes() == b.claims.tobytes()) for a, b in zip(steps, again))
