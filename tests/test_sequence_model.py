"""CPU suite: the sequence model that tests/test_gpu_sequences.py compares every context path with.

The model (tests/sequences.py) carries the library's state across a long sequence of calls with the C oracle.  Here it is
replayed step by step by the pure-Python restatement (oracle/naive.py, plus Deallocate and UnsuitableNodes written from
spec §8/§9 below), and the spec's invariants of the state are checked after every step."""
import copy

import numpy as np
import pytest

import sequences as S
from oracle import naive

KINDS = {"alloc", "error", "sorted", "sorted_bad", "dealloc", "unsuitable", "pods", "selectors", "table", "reset",
         "set_inventory", "calibrate", "idle", "restart"}


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

    def step(self, i, s):
        t = _table(self.inv.tables[self.table])
        claims = None if s.claims is None else _dicts(s.claims)
        off = None if s.out_off is None else [int(x) for x in s.out_off]
        if s.kind in ("alloc", "sorted"):
            if s.flags & S.F_FRESH:
                self.live = copy.deepcopy(self.pristine)
                self.held = {}
            out, after = naive.allocate(self.live, self.off, t, claims, off)
            self.live = [dict(g, node=g0["node"], rsvd=g0["rsvd"]) for g, g0 in zip(after, self.live)]
            self.held[i] = (claims, off, out)
            return out
        if s.kind == "pods":
            out, after = naive.allocate_pods(self.live, self.off, t, claims, [int(x) for x in s.pod_off],
                                             bool(s.flags & S.F_EXHAUSTIVE), off)
            self.live = [dict(g, node=g0["node"], rsvd=g0["rsvd"]) for g, g0 in zip(after, self.live)]
            self.held[i] = (claims, off, out)
            return out
        if s.kind == "dealloc":
            for b in s.batches:
                self.dealloc(*self.held.pop(b))
        elif s.kind == "unsuitable":
            pod_off = [int(x) for x in s.pod_off]
            if s.cand_nodes is None:
                n_pod = len(pod_off) - 1
                cn, co = list(range(self.n_node)) * n_pod, [p * self.n_node for p in range(n_pod + 1)]
            else:
                cn, co = [int(x) for x in s.cand_nodes], [int(x) for x in s.cand_off]
            return self.unsuitable(claims, pod_off, cn, co, bool(s.flags & S.F_EXHAUSTIVE), t)
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


@pytest.mark.parametrize("n_node,seed", [(2, 1), (3, 2), (5, 3), (7, 4), (4, 5), (6, 6)])
def test_model_matches_naive_replay(oracle, n_node, seed):
    """About 30 steps on a small inventory: every output and every state of the model equals the naive replay."""
    inv = _small(n_node, seed)
    steps = S.make_sequence(inv, 30, seed, max_claims=24, selectors=False, calibrate=False)
    S.Model(inv, oracle).run(steps)
    nv = Naive(inv)
    for i, s in enumerate(steps):
        got = nv.step(i, s)
        if s.kind in ("alloc", "sorted", "pods"):
            assert _tuples(s.expect) == got, f"step {i} {s.kind}: OutRecs differ"
        elif s.kind == "unsuitable":
            want = np.packbits(np.array(got, dtype=np.uint8), bitorder="little") if got else np.zeros(0, np.uint8)
            assert s.expect.tobytes() == want.tobytes(), f"step {i}: UnsuitableNodes bits differ"
        assert _state(_dicts(s.live_after)) == _state(nv.live), f"step {i} {s.kind}: state differs"


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
        live = [k for k, (c, off, out, _) in m.held.items() if (out["status"] == 0).any()]
        if live:
            del m.held[live[0]]
            with pytest.raises(AssertionError):
                m.check_invariants()
            return
    pytest.fail("no batch placed anything")


@pytest.mark.parametrize("n_node", [61, 132])
def test_sequence_covers_every_step_kind(n_node):
    """The GPU sequences' shape: every step kind, the sizes at the staged capacity and twice it in OutRecs (each side of
    them), odd OutRec counts, sizes off the 256-claim piece, FRESH and out_off both ways, runs of three or more Allocate
    batches of one shape for a captured graph to replay, and Allocate batches in a row for the resident kernel."""
    w = S.synth.mixed(10, n_node, 40)
    inv = S.inventory("cover", w.gpus, w.node_off, w.table, 40)
    steps = S.make_sequence(inv, 400, 7)
    assert {s.kind for s in steps} == KINDS
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
