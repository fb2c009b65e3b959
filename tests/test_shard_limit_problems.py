"""CPU suite: tests/test_gpu_shard_limits.py tests what it claims.  With the C oracle on the exact problems, splits and
paddings of tests/shard_limit_problems.py:
  - the shard model holds: each rank answers the claims of its node range plus, on the stray rank, the claims naming no
    node; k_shard_compact's slot rule is records.claim_slots in both slot forms and the ranks' totals make n_out; the
    per-rank oracle answers merged by shard.merge are the whole batch's answer
  - the fixed examples reach the limits on a rank that is neither rank 0 nor the stray rank (starts 15, sizes 16, GPU
    claims of count 32 with their 32 slots, co-location runs of 32 and 33 members, every status 0-5), the stray rank answers INVALID GPU claims
    of count 0 and 33 in both slot forms, and the paddings put kept members of one run on both sides of a tile boundary."""
import numpy as np
import pytest

import limit_problems as LP
import shard_limit_problems as SP
from test_gpu_limits import N_EX, ONE_WAVE_FUSED_MAX
from test_gpu_paths import STAGED_CAP
from shard_world import kept as _kept

R = SP.R


@pytest.fixture(scope="module")
def answers(oracle):
    """every form-a problem with the oracle's answer in both slot forms"""
    return [(w, {slot: oracle.allocate(w.gpus, w.node_off, w.table, w.claims, *SP.slot_form(w, slot))[0]
                 for slot in ("off", "nooff")}) for w in SP.problems()]


def test_shard_model_holds(pkg, oracle, answers):
    for w, ans in answers:
        for world, bounds, stray in SP.splits(w):
            what = f"{w.name}, bounds {bounds}, strays on {stray}"
            own = SP.owner(w.claims, w.n_node, bounds, stray)
            for r in range(world):
                assert ((own == r) == _kept(w, bounds[r], bounds[r + 1], r == stray)).all(), f"{what}: rank {r}"
            for have_off, n_out in ((True, w.n_out), (False, w.n_claim)):
                sl = SP.kernel_slots(w.claims, w.n_node, have_off)
                assert (sl == R.claim_slots(w.claims, w.n_node, have_off)).all(), what
                assert sum(int(sl[own == r].sum()) for r in range(world)) == n_out, what
            ranges = [(bounds[r], bounds[r + 1]) for r in range(world)]
            parts = []
            for r in range(world):                       # (shard.local_batch gives the strays to rank 0)
                lb = pkg.shard.local_batch(w.gpus, w.node_off, w.claims, r, ranges)
                out, _ = oracle.allocate(lb.gpus, lb.node_off, w.table, lb.claims, lb.out_off, lb.n_out)
                parts.append((lb.sel, lb.out_off, out, lb.gpu_base))
            assert pkg.shard.merge(w.n_out, w.out_off, parts).tobytes() == ans["off"].tobytes(), what


def _node_runs(w):
    """{node: lengths of its co-location runs, plus 33 where 33 consecutive claims share a group}"""
    res = {}
    for n in range(w.n_node):
        q = list(np.nonzero(w.claims["node"] == n)[0])
        ln = {k for _, k in LP._runs(w.claims, q)}
        c = w.claims
        for k in range(len(q) - 32):
            if all(c[q[k + j]]["kind"] == R.KIND_MIG and c[q[k + j]]["group"] == c[q[k]]["group"] != 0 for j in range(33)):
                ln.add(33)
        res[n] = ln
    return res


@pytest.mark.skipif(N_EX > 0, reason="random seeds (DRA_PROP_EXAMPLES) need not reach every limit")
def test_fixed_examples_reach_the_limits(answers):
    reached, stray_invalid = set(), set()
    for w, ans in answers:
        runs = _node_runs(w)
        node = w.claims["node"].astype(np.int64)
        for world, bounds, stray in SP.splits(w):
            own = SP.owner(w.claims, w.n_node, bounds, stray)
            for slot, out in ans.items():
                oo = w.out_off if slot == "off" else np.arange(w.n_claim)
                sl = SP.kernel_slots(w.claims, w.n_node, slot == "off")
                for r in range(world):
                    for i in np.nonzero(own == r)[0]:
                        x, recs = w.claims[i], out[int(oo[i]): int(oo[i]) + int(sl[i])]
                        if r == stray:
                            if x["kind"] == R.KIND_GPU and x["count"] in (0, 33) and node[i] < w.n_node and \
                                    (recs["status"] == R.ST_INVALID).all():
                                stray_invalid.add((int(x["count"]), slot))
                            continue
                        if r == 0:
                            continue
                        ok = recs["status"] == R.ST_OK
                        reached |= {f"status {s}" for s in recs["status"].tolist()}
                        if (ok & (recs["start"] == 15)).any():
                            reached.add("start 15")
                        if (ok & (recs["size"] == 16)).any():
                            reached.add("size 16")
                        if x["kind"] == R.KIND_GPU and x["count"] == 32 and len(recs) == 32:
                            reached.add("gpu count 32")         # (placed whole by the gpu32 packet fixture)
                        reached |= {f"run {k}" for k in runs.get(int(node[i]), ()) if k in (32, 33)}
    want = {f"status {s}" for s in range(6)} | {"start 15", "size 16", "gpu count 32", "run 32", "run 33"}
    assert want <= reached, sorted(want - reached)
    assert {(0, "off"), (33, "off"), (0, "nooff"), (33, "nooff")} <= stray_invalid, sorted(stray_invalid)


@pytest.mark.parametrize("n_total", [STAGED_CAP + 1, ONE_WAVE_FUSED_MAX + 1, 262_145, 2_097_153])
def test_paddings_straddle_tile_boundaries(n_total):
    """Form b keeps exactly the problem's claims, in order, and some run's kept members lie on both sides of a boundary of
    the compaction's tile (256 claims up to 262,144, 2,048 beyond), with dropped claims between them."""
    probs = SP.problems()
    straddles = 0
    for w in probs[:6] if n_total > 1 << 20 else probs:
        v = SP.padded(w, n_total)
        assert v.tile == (256 if n_total <= 262_144 else 2048)
        keep = _kept(v, v.lo, v.hi, True)
        assert np.nonzero(keep)[0].tolist() == v.pos.tolist()
        assert v.claims[keep].tobytes() == SP.behind_empty_node(w).claims.tobytes()
        assert v.node_off[1] == 0 and v.hi == v.n_node - 1
        for n in range(v.lo, v.hi):
            q = np.nonzero(v.claims["node"] == n)[0]
            for k, ln in LP._runs(v.claims, list(q)):
                p = q[k: k + ln]
                if ln > 1 and len(set((p // v.tile).tolist())) > 1 and (np.diff(p) > 1).all():
                    straddles += 1
    assert straddles, f"no run straddles a {n_total}-claim padding's tile boundary"


def test_every_padding_keeps_the_problem_in_order():
    """The paddings of the chain test of the one-CTA sort and of the selector problems."""
    cases = [(w, SP.SORT_CHAIN_PAD(w)) for w in SP.problems()] + \
            [(SP.selector_problem(s), n) for s in SP.SEL_SEEDS for n in (STAGED_CAP + 1, 262_145, 2_097_153)]
    for w, n_total in cases:
        v = SP.padded(w, n_total)
        assert v.n_claim == n_total and (v.n_claim <= 8192) == (n_total <= 8192)
        keep = _kept(v, v.lo, v.hi, True)
        assert np.nonzero(keep)[0].tolist() == v.pos.tolist(), w.name
        assert v.claims[keep].tobytes() == SP.behind_empty_node(w).claims.tobytes(), w.name


def test_selector_problems_reach_the_claim_beyond_the_table(oracle):
    """Every selector problem's GPU claim of count 3 naming the id past the table keeps three slots, all INVALID; it sits
    on a rank other than the stray rank in some split of every world above 1."""
    for seed in SP.SEL_SEEDS:
        w = SP.selector_problem(seed)
        oracle.set_selectors(w.attrs, w.sels)
        try:
            ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
        finally:
            oracle.set_selectors()
        o = int(w.out_off[w.beyond])
        assert int(w.out_off[w.beyond + 1]) == o + 3 and (ref["status"][o: o + 3] == R.ST_INVALID).all()
        assert int(w.claims["mem_limit_mib"][w.beyond]) == len(w.sels) + 1
        for world in (2, 3, 4):
            assert any(int(SP.owner(w.claims[w.beyond: w.beyond + 1], w.n_node, b, s)[0]) != s
                       for k, b, s in SP.selector_splits(w) if k == world), (seed, world)


@pytest.mark.parametrize("name", SP.PACKET_FIXTURES)
def test_packet_fixtures(oracle, name):
    """Each fixture's records touch the top of the packet field it is named for, on the last rank at worlds 2 and 4."""
    w = SP.packet_fixture(name)
    ref, _ = oracle.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
    assert SP.PACKET_EXPECT[name](ref), ref
    for world in (2, 4):
        own = SP.owner(w.claims, w.n_node, [0] * world + [1], 0)
        assert set(own.tolist()) == {0, world - 1}
