"""CPU suite: a model of the sharded place pods with reasons (dra_place_pods_why_batch_global_device, spec §18 "Sharded
form"): tests/test_place_shard_model.py's protocol with every visit answered.

Each rank walks the visit lists of its own nodes with one cursor per node and a REPLICA of every pod's state word, as
k_pods_place<4, true, true> does; publications reach the peers' replicas late and out of order, and deliveries of one
call may arrive during the next.  A visit that finds its pod's word DONE with a node is a dry run on the node as it
stands: OK on the node the word names, else the reason of §12's steps (place_why_oracle.naive_pod_reason); a PL_NOWHERE
word is skipped.  The reasons go to the rank's slice at the walk index (dense: pod * window width + window node; candidate
form: the pair's index), the prep adds the window's pairs of empty (OK) and over-32-claim (INVALID) pods, and the merge
takes each pair from the rank that owns its node (a candidate naming no node: NO_NODE) and sums the tallies.  After each
call of a run, every output must equal tests/place_why_oracle.py's on the world's state, and placement the §13 oracle's.
Each rank's copy of the GPUs outside its range is wrong on purpose: no rank may read it."""
import copy
import random

import numpy as np
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle import naive as N
from test_oracle_properties import _dicts
from test_place_pods import _flat, place_problems, placed_offsets
from test_place_shard_model import DONE, LIMIT, NOWHERE, POS, Rank
from test_pod_mode import _tbl

import place_why_oracle as PW
import why_oracle as Y


def _run_call(rng, ranks, seq, node_off, table, claims, pod_off, cands, dense, exhaustive, out_off, pending):
    """One call on every rank; returns (pod_node, pair_why, pair_claim, pod_why, claim_blocks) after the merge."""
    n_node, n_pod = len(node_off) - 1, len(pod_off) - 1
    lists = {n: [] for n in range(n_node)}
    for p in range(n_pod):
        for j, n in enumerate(cands[p]):
            if n < n_node:
                lists[n].append((p, j))
    pair0 = [0]
    for p in range(n_pod):
        pair0.append(pair0[-1] + len(cands[p]))

    def walk_index(rk, p, j, n):
        return p * (rk.hi - rk.lo) + (n - rk.lo) if dense else pair0[p] + j

    for rk in ranks:
        rk.prepared = False
        rk.cursor = {n: 0 for n in range(rk.lo, rk.hi)}
        rk.slice = {}

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
            if not live:                                 # the pairs no walk reaches, on this rank's window
                for j, n in enumerate(cands[p]):
                    if rk.lo <= n < rk.hi:
                        rk.slice[walk_index(rk, p, j, n)] = (Y.ST_INVALID if cnt else Y.ST_OK, Y.WHY_CLAIM_NONE)
        rk.prepared = True

    def reason(rk, q, n):
        c0, c1 = pod_off[q], pod_off[q + 1]
        pod = [dict(claims[i], node=n) for i in range(c0, c1)]
        r, b = PW.naive_pod_reason(N, copy.deepcopy(rk.G[node_off[n]:node_off[n + 1]]), table, pod, n_node, exhaustive, True)
        return r, Y.WHY_CLAIM_NONE if b is None else c0 + b

    def step(rk, n):
        lst, c = lists[n], rk.cursor[n]
        if c >= len(lst):
            return False
        q, k = lst[c]
        v = rk.rep[q]
        assert v >> 32 == seq, "a word of another call reached the walk"
        s = v & 0xFFFFFFFF
        if s & DONE:
            if s != NOWHERE:                             # a dry run: the pod was placed at an earlier position
                rk.slice[walk_index(rk, q, k, n)] = (Y.ST_OK, Y.WHY_CLAIM_NONE) if s & ~DONE == n else reason(rk, q, n)
            rk.cursor[n] += 1
            return True
        if (s & POS) > k:
            rk.cursor[n] += 1
            return True
        if (s & POS) < k:
            return False
        r, b = reason(rk, q, n)
        rk.slice[walk_index(rk, q, k, n)] = (r, b)
        c0, c1 = pod_off[q], pod_off[q + 1]
        pod = [dict(claims[i], node=n) for i in range(c0, c1)]
        placed, recs = N.eval_pod(rk.G, node_off[n], node_off[n + 1], table, pod, n_node, exhaustive, True)
        assert placed == (r == Y.ST_OK), "the reason and the evaluation disagree"
        lim = (s & LIMIT) | (LIMIT if r == Y.ST_SEARCH_LIMIT else 0)
        if placed:
            publish(rk, q, DONE | n)
        else:
            nxt = next((j for j in range(k + 1, len(cands[q])) if cands[q][j] < n_node), None)
            publish(rk, q, NOWHERE if nxt is None else nxt | lim)
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
        for kind, rk, n in actions:
            if kind == "prep":
                prep(rk); moved = True
            elif step(rk, n):
                moved = True
            while pending and rng.random() < 0.4:
                r, p, v = pending.pop(rng.randrange(len(pending)))
                ranks[r].rep[p] = max(ranks[r].rep[p], v)
                moved = True
        if not moved and pending:
            r, p, v = pending.pop(rng.randrange(len(pending)))
            ranks[r].rep[p] = max(ranks[r].rep[p], v)
            moved = True
        assert moved, "deadlock: every node waits and nothing is in flight"
    # the merge: each pair from the slice of the rank owning its node, the tallies over the merged pairs
    pod_node, why, blk = [], [], []
    pod_why = [[0] * Y.WHY_N for _ in range(n_pod)]
    blocks = [0] * len(claims)
    for p in range(n_pod):
        w = ranks[0].rep[p] & 0xFFFFFFFF
        assert all(rk.rep[p] == ranks[0].rep[p] for rk in ranks)
        pod_node.append(w & ~DONE if w != NOWHERE else NOWHERE)
        for j, n in enumerate(cands[p]):
            if n >= n_node:
                r, b = Y.WHY_NO_NODE, Y.WHY_CLAIM_NONE
            else:
                owner = next(rk for rk in ranks if rk.lo <= n < rk.hi)
                r, b = owner.slice[walk_index(owner, p, j, n)]
            why.append(r); blk.append(b)
            pod_why[p][r] += 1
            if b != Y.WHY_CLAIM_NONE:
                blocks[b] += 1
    return pod_node, why, blk, pod_why, blocks


@settings(max_examples=120, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(place_problems(), st.booleans(), st.integers(1, 5), st.data())
def test_protocol_with_reasons_equals_the_oracle(pkg, prob, exhaustive, world, data):
    R = pkg.records
    g, off, t, c, pod_off, cands, dense = prob
    n_node = len(off) - 1
    if len(c) and data.draw(st.booleans()):              # an empty pod and one of 33 claims, which no walk reaches
        c = np.concatenate([c, np.repeat(c[:1], 33)])
        pod_off = np.concatenate([pod_off, [pod_off[-1], pod_off[-1] + 33]]).astype(np.uint32)
        extra = [0, n_node + 1, max(n_node - 1, 0), 0]
        cands = list(cands) + [extra, extra[::-1]]
    n_pod = len(pod_off) - 1
    if dense:
        cands = [list(range(n_node)) for _ in range(n_pod)]
    cuts = sorted(data.draw(st.lists(st.integers(0, n_node), min_size=world - 1, max_size=world - 1)))
    bounds = [0] + cuts + [n_node]
    n_calls = data.draw(st.integers(1, 3))
    rng = random.Random(data.draw(st.integers(0, 2 ** 31)))
    out_off, n_out = placed_offsets(R, c, n_node)
    table, claims = _tbl(t), _dicts(c)
    offs, po = [int(x) for x in off], [int(x) for x in pod_off]
    ranks = []
    for r in range(world):                               # a copy that is wrong outside the rank's own GPUs
        mine = g[::-1].copy()
        a, b = offs[bounds[r]], offs[bounds[r + 1]]
        mine[a:b] = g[a:b]
        ranks.append(Rank(r, bounds[r], bounds[r + 1], _dicts(mine), n_pod))
    pending = []
    state = g.copy()
    cn, co = _flat(cands)
    for call in range(1, n_calls + 1):
        ref = PW.place_why(state, off, t, c, pod_off, None if dense else cn, None if dense else co, out_off, n_out,
                           Y.F_EXHAUSTIVE if exhaustive else 0)
        pod_node, why, blk, pod_why, blocks = _run_call(rng, ranks, call, offs, table, claims, po, cands, dense, exhaustive,
                                                        [int(x) for x in out_off], pending)
        assert pod_node == [int(x) for x in ref[1]], f"call {call}: pod_node"
        assert why == [int(x) for x in ref[3]], f"call {call}: pair_why"
        assert blk == [int(x) for x in ref[4]], f"call {call}: pair_claim"
        assert pod_why == [[int(x) for x in row] for row in ref[5]], f"call {call}: pod_why"
        assert blocks == [int(x) for x in ref[6]], f"call {call}: claim_blocks"
        for rk in ranks:                                 # each rank's own GPUs are the world's state
            now = N._dump(None, rk.G)
            for gi in range(offs[rk.lo], offs[rk.hi]):
                a = ref[2][gi]
                assert (int(a["busy"]), int(a["flags"]), int(a["mem_free_mib"]), int(a["share_cnt"])) == \
                    (now[gi]["busy"], now[gi]["flags"], now[gi]["mem_free_mib"], now[gi]["share_cnt"]), f"call {call}: gpu {gi}"
        state = ref[2]
