"""CPU suite: a model of the sharded place-pods protocol (dra_place_pods_batch_global_device, spec §13 "Sharded form").

Each rank walks the visit lists of its own nodes with one cursor per node, exactly as k_pods_place<4, true> does, and
keeps a REPLICA of every pod's 64-bit state word {call sequence : position | LIMIT | DONE}.  A publication goes into the
rank's own replica at once and to every peer's replica as a delivery that is delayed and reordered at random; every
replica merges by max.  Ranks prepare each call at a random moment, so a peer's words of the current call can reach a
rank before its own initial words, and deliveries of a finished call can arrive during the next.  The schedule of ranks
and nodes is random but fair.  After each call of a run, every pod's final word must be DONE on every rank, the records
each pod's finaliser wrote, pod_node and every rank's own node range must equal tests/place_oracle.py's sequential rule
on the world's state, and no schedule may deadlock.  Pods are evaluated with oracle/naive.py's pod evaluation."""
import random

from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle import naive as N
from test_oracle_properties import _dicts
from test_place_pods import _flat, place_problems, placed_offsets
from test_pod_mode import _tbl

import place_oracle as P

DONE, LIMIT, POS, NOWHERE = 0x80000000, 0x40000000, 0x3FFFFFFF, 0xFFFFFFFF


class Rank:
    def __init__(self, r, lo, hi, gpus, n_pod):
        self.r, self.lo, self.hi = r, lo, hi
        self.G = N._state(gpus)              # this rank's inventory copy: authoritative for its own nodes only
        self.rep = [0] * n_pod               # the replica of every pod's state word
        self.prepared = False
        self.cursor = {}


def _run_call(rng, ranks, bounds, seq, node_off, table, claims, pod_off, cands, exhaustive, out_off, pending):
    """One call of the protocol on every rank; returns (the records the finalisers wrote, by slot; pod_node)."""
    n_node, n_pod = len(node_off) - 1, len(pod_off) - 1
    lists = {n: [] for n in range(n_node)}   # node -> its visits (pod, position) in the order the sequential rule makes them
    for p in range(n_pod):
        for j, n in enumerate(cands[p]):
            if n < n_node:
                lists[n].append((p, j))
    for rk in ranks:
        rk.prepared = False
        rk.cursor = {n: 0 for n in range(rk.lo, rk.hi)}
    records = {}                             # slot -> record, as the finalisers wrote them
    pod_node = [NOWHERE] * n_pod

    def slots_of(i):
        return N._slots(dict(claims[i], node=0), 1, True)

    def fail_records(p, st_):
        for i in range(pod_off[p], pod_off[p + 1]):
            inv = len(claims[pod_off[p]:pod_off[p + 1]]) > N.MAX_POD or N._invalid(dict(claims[i], node=0), 1, True)
            for k in range(slots_of(i)):
                records[out_off[i] + k] = (NOWHERE, 0, 0, N._oprof(claims[i]), 5 if inv else st_)

    def publish(rk, p, word):
        v = (seq << 32) | word
        rk.rep[p] = max(rk.rep[p], v)
        for other in ranks:
            if other is not rk:
                pending.append((other.r, p, v))

    def prep(rk):
        for p in range(n_pod):
            cnt = pod_off[p + 1] - pod_off[p]
            live = 0 < cnt <= N.MAX_POD
            first = next((j for j, n in enumerate(cands[p]) if n < n_node), None)
            w = first if live and first is not None else NOWHERE
            rk.rep[p] = max(rk.rep[p], (seq << 32) | w)
            if cnt and w == NOWHERE:         # never evaluated: every rank writes the same records
                fail_records(p, 6)
        rk.prepared = True

    def step(rk, n):
        """One entry of node n's list on rank rk; True when the cursor moved."""
        lst, c = lists[n], rk.cursor[n]
        if c >= len(lst):
            return False
        q, k = lst[c]
        v = rk.rep[q]
        assert v >> 32 == seq, "a word of another call reached the walk"
        s = v & 0xFFFFFFFF
        if s & DONE or (s & POS) > k:
            rk.cursor[n] += 1
            return True
        if (s & POS) < k:
            return False                     # q may still come here: the node waits
        c0, c1 = pod_off[q], pod_off[q + 1]
        pod = [dict(claims[i], node=n) for i in range(c0, c1)]
        placed, recs = N.eval_pod(rk.G, node_off[n], node_off[n + 1], table, pod, n_node, exhaustive, True)
        lim = (s & LIMIT) | (LIMIT if any(r[0][4] == 7 for r in recs if r) else 0)
        if placed:
            for i, r in zip(range(c0, c1), recs):
                for k_, rec in enumerate(r):
                    records[out_off[i] + k_] = rec
            publish(rk, q, DONE | n)
        else:
            nxt = next((j for j in range(k + 1, len(cands[q])) if cands[q][j] < n_node), None)
            if nxt is None:
                fail_records(q, 7 if lim else 6)
                publish(rk, q, NOWHERE)
            else:
                publish(rk, q, nxt | lim)
        rk.cursor[n] += 1
        return True

    def finished(rk):
        return rk.prepared and all(rk.cursor[n] >= len(lists[n]) for n in rk.cursor) and \
            all(v >> 32 == seq and v & DONE for v in rk.rep)

    while not all(finished(rk) for rk in ranks):
        actions = []
        for rk in ranks:
            if not rk.prepared:
                actions.append(("prep", rk, None))
            else:
                actions += [("walk", rk, n) for n in rk.cursor if rk.cursor[n] < len(lists[n])]
        rng.shuffle(actions)
        moved = False
        for kind, rk, n in actions:          # fair: every enabled action is tried once a round, in a random order
            if kind == "prep":
                prep(rk); moved = True
            elif step(rk, n):
                moved = True
            while pending and rng.random() < 0.4:            # some deliveries, in a random order, between the steps
                r, p, v = pending.pop(rng.randrange(len(pending)))
                ranks[r].rep[p] = max(ranks[r].rep[p], v)
                moved = True
        if not moved and pending:
            r, p, v = pending.pop(rng.randrange(len(pending)))
            ranks[r].rep[p] = max(ranks[r].rep[p], v)
            moved = True
        assert moved, "deadlock: every node waits and nothing is in flight"
    for p in range(n_pod):
        w = ranks[0].rep[p] & 0xFFFFFFFF
        assert all(rk.rep[p] == ranks[0].rep[p] for rk in ranks)
        pod_node[p] = w & ~DONE if w != NOWHERE else NOWHERE
    return records, pod_node


@settings(max_examples=150, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(place_problems(), st.booleans(), st.integers(1, 4), st.data())
def test_protocol_equals_sequential_rule(pkg, prob, exhaustive, world, data):
    R = pkg.records
    g, off, t, c, pod_off, cands, dense = prob
    n_node, n_pod = len(off) - 1, len(pod_off) - 1
    if dense:
        cands = [list(range(n_node)) for _ in range(n_pod)]
    cuts = sorted(data.draw(st.lists(st.integers(0, n_node), min_size=world - 1, max_size=world - 1)))
    bounds = [0] + cuts + [n_node]
    n_calls = data.draw(st.integers(1, 3))
    rng = random.Random(data.draw(st.integers(0, 2 ** 31)))
    out_off, n_out = placed_offsets(R, c, n_node)
    table, claims = _tbl(t), _dicts(c)
    offs, po, oo = [int(x) for x in off], [int(x) for x in pod_off], [int(x) for x in out_off]
    ranks = [Rank(r, bounds[r], bounds[r + 1], _dicts(g), n_pod) for r in range(world)]
    pending = []                             # deliveries in flight, carried from one call into the next
    state = g.copy()
    cn, co = _flat(cands)
    for call in range(1, n_calls + 1):
        ref, ref_node, ref_after = P.place_pods(state, off, t, c, pod_off, cn, co, out_off, n_out,
                                                P.F_EXHAUSTIVE if exhaustive else 0)
        records, pod_node = _run_call(rng, ranks, bounds, call, offs, table, claims, po, cands, exhaustive, oo, pending)
        assert [int(x) for x in pod_node] == [int(x) for x in ref_node], f"call {call}: pod_node"
        for s in range(int(n_out)):
            want = tuple(int(v) for v in ref[s])
            if want != (0, 0, 0, 0, 0):
                assert records.get(s) == want, f"call {call}: slot {s}"
        for rk in ranks:                     # each rank's own GPUs are the world's state
            mine = N._dump(None, rk.G)
            for gi in range(offs[rk.lo], offs[rk.hi]):
                a = ref_after[gi]
                assert (int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) == \
                    (mine[gi]["busy"], mine[gi]["flags"], mine[gi]["mem_free_mib"], mine[gi]["share_cnt"]), f"call {call}: gpu {gi}"
        state = ref_after
