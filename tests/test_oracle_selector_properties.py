"""CPU suite: property-based pinning of the selector semantics (spec §10).

An independent Python evaluator of the postfix predicate programs decides, per GPU, whether it passes a randomly
drawn selector (malformed programs included).  Spec §10 says a GPU that fails the claim's selector "is simply not
eligible (and, for MIG, does not offer the profile)" — exactly what the UNAVAILABLE flag means — so a batch whose
claims all carry selector s must allocate exactly like the selector-free batch on an inventory where the failing
GPUs are flagged UNAVAILABLE.  The right-hand side is the selector-free oracle, itself cross-checked by
oracle/naive.py in test_oracle_properties.py."""
import numpy as np
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from test_oracle_properties import problems


def sel_eval(prog, a):
    """spec §10, restated: postfix program over a boolean stack; empty = true; underflow / unknown code = false."""
    stack, seen = [], False
    for ins in prog:
        op = int(ins["op"])
        if op == 0:
            break
        seen = True
        if op == 1:
            attr, cmp_, val = int(ins["attr"]), int(ins["cmp"]), int(ins["value"])
            if attr > 4:
                return False
            v = int([a["mem_total_mib"], a["cc"], a["index"], a["product"], a["driver_major"]][attr])
            if cmp_ > 6:
                return False
            stack.append([v == val, v != val, v < val, v <= val, v > val, v >= val, v < 32 and (val >> v) & 1 == 1][cmp_])
        elif op in (2, 3):
            if len(stack) < 2:
                return False
            b, a_ = stack.pop(), stack.pop()
            stack.append((a_ and b) if op == 2 else (a_ or b))
        elif op == 4:
            if not stack:
                return False
            stack.append(not stack.pop())
        else:
            return False
    return stack[-1] if seen else True


def selector_programs(D, n_gpu):
    """Random attributes for n_gpu GPUs, a table of 1-3 random selector programs and a selector id (the table's size + 1:
    beyond it).  D draws integers and picks (preempt_problems._Hyp from hypothesis, _Rng from a seeded generator)."""
    import importlib
    R = importlib.import_module("k8s-dra-driver_b200").records
    a = np.zeros(n_gpu, dtype=R.ATTR_DTYPE)
    for i in range(n_gpu):
        a[i] = (D.pick([16384, 40960, 81920]), D.pick([0x0705, 0x0800, 0x0900]), D.int(0, 9), D.int(0, 5),
                D.pick([535, 550, 570]))
    n_sel = D.int(1, 3)
    sels = np.zeros((n_sel, R.SEL_MAX_INS), dtype=R.SEL_INS_DTYPE)
    domain = {0: [16384, 40960, 81920], 1: [0x0705, 0x0800, 0x0900], 2: list(range(10)), 3: list(range(6)), 4: [535, 550, 570]}

    def leaf():
        attr = D.int(0, 4)
        if attr in (2, 3) and D.int(0, 1):
            return [(1, attr, 6, 0, D.int(0, 1023))]                         # IN_MASK over small ids
        return [(1, attr, D.int(0, 5), 0, D.pick(domain[attr]))]

    def tree(depth):
        if depth == 0 or D.int(0, 2) == 0:
            return leaf()
        k = D.pick([2, 3, 4])
        if k == 4:
            return tree(depth - 1) + [(4, 0, 0, 0, 0)]
        return tree(depth - 1) + tree(depth - 1) + [(k, 0, 0, 0, 0)]

    for s in range(n_sel):
        if D.int(0, 4) != 0:                               # mostly well-formed trees that split the GPUs ...
            prog = tree(2)[: R.SEL_MAX_INS]
            for k, ins in enumerate(prog):
                sels[s, k] = ins
        else:                                              # ... and some garbage: unknown codes, underflow, early END
            for k in range(D.int(0, R.SEL_MAX_INS)):
                sels[s, k] = (D.pick([1, 1, 1, 2, 3, 4, 0, 9]), D.pick([0, 1, 2, 3, 4, 7]), D.pick([0, 1, 2, 3, 4, 5, 6, 8]), 0,
                              D.pick([0, 1, 3, 0b101010, 535, 0x0800, 40960, 0xFFFFFFFF]))
    sid = D.int(1, n_sel + 1)                             # n_sel + 1: beyond the table -> INVALID
    return a, sels, sid


@st.composite
def selector_problems(draw):
    from preempt_problems import _Hyp
    g, off, t, c, out_off, n_out = draw(problems())
    return (g, off, t, c, out_off, n_out) + selector_programs(_Hyp(draw), len(g))


@settings(max_examples=300, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(selector_problems())
def test_selector_equals_marking_failing_gpus_unavailable(pkg, oracle, prob):
    R = pkg.records
    g, off, t, c, out_off, n_out, attrs, sels, sid = prob
    n_node = len(off) - 1
    # every claim carries selector `sid` (GPU / MIG: in mem_limit_mib; SHARED: in group — spec §10)
    cs = c.copy()
    gm = (cs["kind"] == R.KIND_GPU) | (cs["kind"] == R.KIND_MIG)
    cs["mem_limit_mib"] = np.where(gm, sid, cs["mem_limit_mib"])
    cs["group"] = np.where(cs["kind"] == R.KIND_SHARED, sid, cs["group"])
    carries = gm | (cs["kind"] == R.KIND_SHARED)          # claims of an unknown kind carry nothing
    try:
        oracle.set_selectors(attrs, sels)
        out, after = oracle.allocate(g, off, t, cs, out_off, n_out)
    finally:
        oracle.set_selectors()
    slots = R.claim_slots(cs, n_node)
    if sid > len(sels):                                    # unknown id: the claim keeps its slots, all INVALID
        for i in range(len(cs)):
            if carries[i]:
                assert all(out[int(out_off[i]) + k]["status"] == R.ST_INVALID for k in range(int(slots[i])))
        assert after.tobytes() == g.tobytes() or not carries.all()
        return
    passes = np.array([sel_eval(sels[sid - 1], attrs[i]) for i in range(len(g))], dtype=bool)
    # the same batch WITHOUT selectors on an inventory whose failing GPUs are unavailable
    g2 = g.copy()
    g2["flags"] = np.where(passes, g2["flags"], g2["flags"] | R.GPU_UNAVAILABLE)
    c2 = c.copy()
    c2["mem_limit_mib"] = np.where(gm, 0, c2["mem_limit_mib"])        # GPU / MIG claims: the field is unused without a selector
    c2["group"] = np.where(c2["kind"] == R.KIND_SHARED, 0, c2["group"])
    ref_out, ref_after = oracle.allocate(g2, off, t, c2, out_off, n_out)
    assert out.tobytes() == ref_out.tobytes()
    assert (after["busy"] == ref_after["busy"]).all() and (after["mem_free_mib"] == ref_after["mem_free_mib"]).all()
    assert (after["share_cnt"] == ref_after["share_cnt"]).all()
    assert ((after["flags"] | np.where(passes, 0, R.GPU_UNAVAILABLE)) == ref_after["flags"]).all()
    ok = out["status"] == R.ST_OK                         # and, directly: no OK slot on a GPU that fails the selector
    assert passes[out["gpu"][ok]].all()
