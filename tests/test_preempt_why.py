"""CPU suite: spec §19 — why preemption judged each node as it did, for preemption (§14) and for preempt and place (§15).

The two statements of tests/preempt_why_oracle.py (the C oracles' statuses with place_why_oracle.pair_reason, and the
naive restatement on preempt_naive / preempt_place_naive and naive_pod_reason) share no code; agreement between them pins
the rule.  Then the consequences §19 lists, the tallies, and the two worked examples of the spec."""
import importlib

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings

from preempt_problems import I32_MIN, place_problems, problems
from test_oracle_properties import _dicts
from test_pod_mode import _tbl
from test_preempt import _outs

import place_why_oracle as PW
import preempt_oracle as P
import preempt_place_oracle as PP
import preempt_why_oracle as PY
import why_oracle as Y
from oracle import oracle as O

R = importlib.import_module("k8s-dra-driver_b200").records
NONE = 0xFFFFFFFF


def _args(pb):
    cn, co = pb.cand_arrays()
    return (pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, pb.prio, pb.run_claims, pb.run_pod_off, pb.run_prio,
            pb.run_out, pb.run_out_off, cn, co)


def _naive_args(pb):
    return (_dicts(pb.gpus), [int(x) for x in pb.node_off], _tbl(pb.table), _dicts(pb.claims),
            [int(x) for x in pb.pod_off], [int(x) for x in pb.prio], pb.cands, bool(pb.flags & P.F_EXHAUSTIVE),
            _dicts(pb.run_claims), [int(x) for x in pb.run_pod_off], [int(x) for x in pb.run_prio], _outs(pb.run_out))


def _same(a, b):
    """the array statement a against the list statement b"""
    assert [int(x) for x in a[0]] == list(b[0]), "pair_status"
    assert [int(x) for x in a[1]] == list(b[1]), "pair_why"
    assert [int(x) for x in a[2]] == list(b[2]), "pair_claim"
    assert a[3].tolist() == [list(r) for r in b[3]] or (not len(a[3]) and not b[3]), "pod_why"
    assert a[4].tolist() == list(b[4]), "claim_blocks"


def _tallies_hold(res, n_pod, pod_off, cand_off, n_node):
    st, why, claim, pod_why, blocks = res
    for p in range(n_pod):
        n = n_node if cand_off is None else int(cand_off[p + 1] - cand_off[p])
        assert int(pod_why[p].sum()) == n
    assert int(blocks.sum()) == int((claim != NONE).sum())
    for k in range(len(why)):                            # consequences 1 and 2
        assert (why[k] == Y.ST_OK) == (st[k] == P.FITS), k
        if st[k] in (P.NO, P.SEARCH_LIMIT):
            assert (why[k] == Y.ST_SEARCH_LIMIT) == (st[k] == P.SEARCH_LIMIT), k
        assert why[k] != Y.ST_GROUP
        if why[k] in (Y.ST_OK, Y.WHY_NO_NODE):
            assert claim[k] == NONE, k
        elif why[k] != Y.ST_INVALID:                     # (INVALID names no claim for a pod of more than 32)
            assert claim[k] != NONE, k


# ---- the two statements agree --------------------------------------------------------------------------------------
@settings(max_examples=60, deadline=None, suppress_health_check=list(HealthCheck))
@given(problems())
def test_preempt_why_statements_agree(pb):
    if pb.error:
        with pytest.raises(ValueError):
            PY.preempt_why(*_args(pb), flags=pb.flags)
        return
    a = PY.preempt_why(*_args(pb), flags=pb.flags)
    b = PY.preempt_why_naive(*_naive_args(pb), None if pb.run_out_off is None else [int(x) for x in pb.run_out_off])
    _same(a, b)
    _tallies_hold(a, len(pb.prio), pb.pod_off, pb.cand_arrays()[1], pb.n_node)
    if not pb.flags & P.F_EXHAUSTIVE:
        assert Y.ST_SEARCH_LIMIT not in a[1]


@settings(max_examples=40, deadline=None, suppress_health_check=list(HealthCheck))
@given(place_problems())
def test_preempt_place_why_statements_agree(pb):
    cn, co = pb.cand_arrays()
    if pb.error:
        with pytest.raises(ValueError):
            PY.preempt_place_why(*_args(pb), pb.out_off, pb.n_out, pb.flags)
        return
    a = PY.preempt_place_why(*_args(pb), pb.out_off, pb.n_out, pb.flags)
    b = PY.preempt_place_why_naive(*_naive_args(pb), None if pb.out_off is None else [int(x) for x in pb.out_off],
                                   None if pb.run_out_off is None else [int(x) for x in pb.run_out_off])
    _same(a[5:], b)
    _tallies_hold(a[5:], len(pb.prio), pb.pod_off, co, pb.n_node)
    # asking for reasons changes nothing §15 defines
    ref = pb.pp_oracle()
    for x, y in zip(a[:5], ref):
        assert x.tobytes() == y.tobytes()


# ---- consequences ----------------------------------------------------------------------------------------------------
@settings(max_examples=40, deadline=None, suppress_health_check=list(HealthCheck))
@given(problems())
def test_consequence_3_against_unsuitable_why(pb):
    """§14 form with DRA_F_EXHAUSTIVE: §17's answer on S, or on S after Deallocate of V for NO / SEARCH_LIMIT pairs with
    a non-empty V"""
    if pb.error:
        return
    cn, co = pb.cand_arrays()
    st, why, claim, _, _ = PY.preempt_why(*_args(pb), flags=P.F_EXHAUSTIVE)
    u_why, u_claim, _, _ = Y.why(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, Y.F_EXHAUSTIVE)
    eff = PY._run_effects(pb.gpus, pb.node_off, pb.run_claims, pb.run_pod_off, pb.run_out, pb.run_out_off)
    lists = PY._cand_lists(len(pb.prio), pb.n_node, cn, co)
    k = 0
    for p, nodes in enumerate(lists):
        for n in nodes:
            V = [r for r in range(len(eff)) if eff[r][0] == n and pb.run_prio[r] < pb.prio[p]]
            if st[k] in (P.NO, P.SEARCH_LIMIT) and V:
                keep = np.zeros(len(pb.run_claims), bool)
                for r in V:
                    keep[pb.run_pod_off[r]:pb.run_pod_off[r + 1]] = True
                if pb.run_out_off is None:
                    g = O.deallocate(pb.gpus, pb.run_claims[keep], pb.run_out[keep], n_node=pb.n_node)
                else:
                    g = O.deallocate(pb.gpus, pb.run_claims[keep], pb.run_out, pb.run_out_off[keep], n_node=pb.n_node)
                w, c, _, _ = Y.why(g, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, Y.F_EXHAUSTIVE)
                assert (why[k], claim[k]) == (w[k], c[k]), (p, n)
            else:
                assert (why[k], claim[k]) == (u_why[k], u_claim[k]), (p, n)
            k += 1


@settings(max_examples=30, deadline=None, suppress_health_check=list(HealthCheck))
@given(place_problems())
def test_consequence_4_host_loop(pb):
    """§15 form with out_off: pod p's records are the §14 form's for that one pod against W_p and the running pods no
    earlier pod evicted"""
    if pb.error or pb.out_off is None:
        return
    cn, co = pb.cand_arrays()
    a = PY.preempt_place_why(*_args(pb), pb.out_off, pb.n_out, pb.flags)
    lists = PY._cand_lists(len(pb.prio), pb.n_node, cn, co)
    k = 0
    for p, nodes in enumerate(lists):
        c0, c1 = int(pb.pod_off[p]), int(pb.pod_off[p + 1])
        pre = PP.preempt_place(pb.gpus, pb.node_off, pb.table, pb.claims[:c0], pb.pod_off[:p + 1], pb.prio[:p],
                               pb.run_claims, pb.run_pod_off, pb.run_prio, pb.run_out, pb.run_out_off,
                               None if co is None else cn[:co[p]], None if co is None else co[:p + 1], pb.out_off[:c0],
                               pb.n_out, pb.flags)
        alive = [r for r in range(len(pb.run_prio)) if pre[3][r] == NONE]
        idx = [i for r in alive for i in range(int(pb.run_pod_off[r]), int(pb.run_pod_off[r + 1]))]
        rpo = np.concatenate([[0], np.cumsum([pb.run_pod_off[r + 1] - pb.run_pod_off[r] for r in alive])]).astype(np.uint32)
        one_claims = pb.claims[c0:c1]
        b = PY.preempt_why(pre[4], pb.node_off, pb.table, one_claims, np.array([0, c1 - c0], np.uint32),
                           pb.prio[p:p + 1], pb.run_claims[idx], rpo, pb.run_prio[alive],
                           pb.run_out if pb.run_out_off is not None else pb.run_out[idx],
                           None if pb.run_out_off is None else pb.run_out_off[idx],
                           None if co is None else np.array(nodes, np.uint32),
                           None if co is None else np.array([0, len(nodes)], np.uint32), pb.flags)
        m = len(nodes)
        assert [int(x) for x in a[5][k:k + m]] == [int(x) for x in b[0]]
        assert [int(x) for x in a[6][k:k + m]] == [int(x) for x in b[1]]
        assert [int(x) for x in a[7][k:k + m]] == [NONE if x == NONE else int(x) + c0 for x in b[2]]
        k += m


@settings(max_examples=40, deadline=None, suppress_health_check=list(HealthCheck))
@given(place_problems())
def test_consequence_5_place_pods_equivalence(pb):
    """no running pod below any pending pod: the reasons are place pods' (§18), byte for byte"""
    if pb.error:
        return
    pb.prio = np.full(len(pb.prio), I32_MIN, np.int32)
    cn, co = pb.cand_arrays()
    a = PY.preempt_place_why(*_args(pb), pb.out_off, pb.n_out, pb.flags)
    b = PW.place_why(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, pb.out_off, pb.n_out, pb.flags)
    for x, y in zip(a[6:], b[3:]):
        assert np.asarray(x).tobytes() == np.asarray(y, x.dtype).tobytes()


# ---- the worked examples of spec §19 ---------------------------------------------------------------------------------
@pytest.fixture
def evict_does_not_help():
    """One node: GPU 0 (non-MIG) fully allocated to a priority-0 pod, GPU 1 (MIG, model 0) fully taken by two 3g pods of
    priority 10.  A priority-5 pod asks for {c0: one full GPU, c1: 3g}."""
    g, off = R.make_inventory([2], mig=True)
    g["flags"][0] = R.GPU_FULL_ALLOCATED
    g["busy"][1] = 0xFF
    rc = np.zeros(3, R.CLAIM_DTYPE)
    ro = np.zeros(3, R.OUT_DTYPE)
    rc["kind"] = [R.KIND_GPU, R.KIND_MIG, R.KIND_MIG]
    rc["profile"] = [0, R.GI_3_SLICE, R.GI_3_SLICE]
    rc["count"] = 1
    for i, (gpu, s, size, prof) in enumerate([(0, 0, 0, R.PROFILE_GPU), (1, 0, 4, R.GI_3_SLICE), (1, 4, 4, R.GI_3_SLICE)]):
        ro[i]["gpu"], ro[i]["start"], ro[i]["size"], ro[i]["profile"], ro[i]["status"] = gpu, s, size, prof, R.ST_OK
    c = np.zeros(2, R.CLAIM_DTYPE)
    c["kind"] = [R.KIND_GPU, R.KIND_MIG]
    c["profile"] = [0, R.GI_3_SLICE]
    c["count"] = 1
    return dict(gpus=g, node_off=off, table=R.default_table(), claims=c, pod_off=np.array([0, 2], np.uint32),
                prio=np.array([5], np.int32), run_claims=rc, run_pod_off=np.arange(4, dtype=np.uint32),
                run_prio=np.array([0, 10, 10], np.int32), run_out=ro)


@pytest.fixture
def lost_to_an_earlier_pod():
    """One MIG GPU of model 0: r0 (priority 10) holds 3g@0, r1 (priority 0) holds 3g@4.  Two pending 3g pods, p0 and
    p1, both of priority 5."""
    g, off = R.make_inventory([1], mig=True)
    g["busy"][0] = 0xFF
    rc = np.zeros(2, R.CLAIM_DTYPE)
    ro = np.zeros(2, R.OUT_DTYPE)
    rc["kind"], rc["profile"], rc["count"] = R.KIND_MIG, R.GI_3_SLICE, 1
    for i, s in enumerate((0, 4)):
        ro[i]["gpu"], ro[i]["start"], ro[i]["size"], ro[i]["profile"], ro[i]["status"] = 0, s, 4, R.GI_3_SLICE, R.ST_OK
    c = np.zeros(2, R.CLAIM_DTYPE)
    c["kind"], c["profile"], c["count"] = R.KIND_MIG, R.GI_3_SLICE, 1
    return dict(gpus=g, node_off=off, table=R.default_table(), claims=c, pod_off=np.array([0, 1, 2], np.uint32),
                prio=np.array([5, 5], np.int32), run_claims=rc, run_pod_off=np.arange(3, dtype=np.uint32),
                run_prio=np.array([10, 0], np.int32), run_out=ro)


@pytest.mark.parametrize("flags", [0, Y.F_EXHAUSTIVE])
def test_evicting_does_not_free_the_mig_claim(evict_does_not_help, flags):
    f = evict_does_not_help
    u_why, u_claim, _, _ = Y.why(f["gpus"], f["node_off"], f["table"], f["claims"], f["pod_off"], flags=Y.F_EXHAUSTIVE)
    assert (int(u_why[0]), int(u_claim[0])) == (Y.ST_NO_CAPACITY, 0)        # §17 names c0 on the live node
    st, why, claim, pod_why, blocks = PY.preempt_why(**f, flags=flags)
    assert (int(st[0]), int(why[0]), int(claim[0])) == (P.NO, Y.ST_NO_CAPACITY, 1)   # §19: c1, which no eviction frees
    assert pod_why[0].tolist() == [0, 1, 0, 0, 0, 0, 0, 0, 0] and blocks.tolist() == [0, 1]


@pytest.mark.parametrize("flags", [0, Y.F_EXHAUSTIVE])
def test_the_second_pod_finds_its_victim_gone(lost_to_an_earlier_pod, flags):
    f = lost_to_an_earlier_pod
    st, why, claim, _, _ = PY.preempt_why(**f, flags=flags)
    assert st.tolist() == [P.EVICT, P.EVICT]                                  # §14 tells both to evict r1
    assert why.tolist() == [Y.ST_NO_CAPACITY] * 2 and claim.tolist() == [0, 1]
    res = PY.preempt_place_why(**f, flags=flags)
    out, pod_node, pod_status, evicted_by = res[:4]
    assert pod_status.tolist() == [P.EVICT, P.NO] and evicted_by.tolist() == [0xFFFFFFFF, 0]
    assert (int(out[0]["start"]), int(out[0]["status"])) == (4, R.ST_OK)
    st, why, claim, pod_why, blocks = res[5:]
    assert st.tolist() == [P.EVICT, P.NO]
    assert why.tolist() == [Y.ST_NO_CAPACITY, Y.ST_NO_CAPACITY] and claim.tolist() == [0, 1]
    assert blocks.tolist() == [1, 1]


def test_never_judged_pods():
    """§15 pairs no judgement reaches: an invalid pod (a 2-GPU claim without out_off), an empty pod, a stray candidate"""
    g, off = R.make_inventory([2, 2], mig=False)
    c = np.zeros(3, R.CLAIM_DTYPE)
    c["kind"], c["count"] = R.KIND_GPU, [1, 2, 1]
    pod_off = np.array([0, 2, 2, 3], np.uint32)
    cn = np.array([0, 7, 1, 5, 0, 1], np.uint32)
    co = np.array([0, 2, 4, 6], np.uint32)
    none = np.zeros(0, R.CLAIM_DTYPE)
    res = PY.preempt_place_why(g, off, R.default_table(), c, pod_off, np.zeros(3, np.int32), none,
                               np.zeros(1, np.uint32), np.zeros(0, np.int32), np.zeros(0, R.OUT_DTYPE), None, cn, co)
    st, why, claim = res[5].tolist(), res[6].tolist(), res[7].tolist()
    assert st == [P.INVALID, P.NO, P.FITS, P.NO, P.FITS, P.FITS]
    assert why == [Y.ST_INVALID, Y.WHY_NO_NODE, Y.ST_OK, Y.WHY_NO_NODE, Y.ST_OK, Y.ST_OK]
    assert claim == [1, NONE, NONE, NONE, NONE, NONE]
