"""CPU suite: spec §14 (preemption) on random problems (tests/preempt_problems.py): mixed node widths, running records that
match the inventory and records perturbed so that they do not, priorities at the int32 ends with many ties, long and
stray-laden candidate lists.  The C oracle must equal the independent restatement (preempt_oracle.preempt_naive), keep
§14's invariants, and on matched records its answer must be one the pods Allocate can carry out."""
import importlib

import numpy as np
from hypothesis import HealthCheck, given, settings

from preempt_problems import NONE, problems
from test_oracle_properties import _dicts
from test_pod_mode import _tbl
from test_preempt import _outs

import preempt_oracle as P

R = importlib.import_module("k8s-dra-driver_b200").records


def _naive(pb):
    return P.preempt_naive(_dicts(pb.gpus), list(pb.node_off), _tbl(pb.table), _dicts(pb.claims), list(pb.pod_off),
                           list(pb.prio), pb.cands, bool(pb.flags & P.F_EXHAUSTIVE), _dicts(pb.run_claims),
                           list(pb.run_pod_off), list(pb.run_prio), _outs(pb.run_out),
                           None if pb.run_out_off is None else [int(x) for x in pb.run_out_off], pb.max_victims)


def _check_invariants(pb, res, oracle):
    pst, pvi, node, st, nv, vic = res
    n_node, mv = pb.n_node, pb.max_victims
    cn, co = pb.cand_arrays()
    for k in range(len(pst)):
        assert pst[k] == P.EVICT or pvi[k] == 0, k
    for p in range(len(pb.prio)):
        row = [int(x) for x in vic[p]]
        n = min(int(nv[p]), mv)
        assert row[n:] == [NONE] * (mv - n)                                   # padded
        assert NONE not in row[:n] and int(nv[p]) >= n
        assert st[p] == P.EVICT or nv[p] == 0
        v = row[:n]
        assert all(pb.run_prio[r] < pb.prio[p] for r in v)                    # strictly lower priority
        keys = [(-int(pb.run_prio[r]), r) for r in v]
        assert keys == sorted(keys) and len(set(v)) == len(v)                 # V order
        if st[p] in (P.FITS, P.EVICT):
            k0 = p * n_node if co is None else int(co[p])
            k1 = k0 + n_node if co is None else int(co[p + 1])
            nodes = list(range(n_node)) if co is None else [int(x) for x in cn[k0:k1]]
            assert node[p] in nodes
            if st[p] == P.EVICT:
                assert any(pst[k] == P.EVICT and pvi[k] == nv[p] for k in range(k0, k1))
        else:
            assert node[p] == NONE
    if pb.flags & P.F_EXHAUSTIVE and len(pst):
        n_pod = len(pb.prio)
        if co is None:
            cn = np.tile(np.arange(n_node, dtype=np.uint32), n_pod)
            co = (np.arange(n_pod + 1) * n_node).astype(np.uint32)
        bits = oracle.unsuitable(pb.gpus, pb.node_off, pb.table, pb.claims, pb.pod_off, cn, co, flags=oracle.F_EXHAUSTIVE)
        fits = np.unpackbits(bits, bitorder="little")[: len(pst)].astype(bool)
        assert (fits == (pst == P.FITS)).all()


def _check_flow(pb, res, oracle):
    """matched records: deallocate the chosen victims, then the pods Allocate places the pod on pod_node"""
    _, _, node, st, nv, _ = res
    full = pb.oracle(max_victims=max(1, int(nv.max(initial=0))))[5]
    roo = pb.run_out_off
    for p in np.flatnonzero((st == P.EVICT) | (st == P.FITS)):
        if pb.pod_off[p + 1] == pb.pod_off[p]:
            continue
        keep = np.zeros(len(pb.run_claims), bool)
        for r in full[p][: nv[p]]:
            keep[pb.run_pod_off[r]: pb.run_pod_off[r + 1]] = True
        if roo is None:
            g = oracle.deallocate(pb.gpus, pb.run_claims[keep], pb.run_out[keep], n_node=pb.n_node)
        else:
            g = oracle.deallocate(pb.gpus, pb.run_claims[keep], pb.run_out, roo[keep], n_node=pb.n_node)
        pod = pb.claims[pb.pod_off[p]: pb.pod_off[p + 1]].copy()
        pod["node"] = node[p]
        oo, n_out = R.out_offsets(pod, pb.n_node)
        out, _ = oracle.allocate_pods(g, pb.node_off, pb.table, pod, np.array([0, len(pod)], np.uint32), oo, n_out,
                                      flags=pb.flags)
        assert (out["status"] == R.ST_OK).all(), (p, st[p])


@settings(max_examples=300, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(problems())
def test_oracle_agrees_with_naive_and_keeps_the_invariants(oracle, pb):
    try:
        res = pb.oracle()
    except ValueError:
        assert pb.error, pb.what                          # only the call-level errors of §14 are refused
        return
    assert not pb.error, pb.what
    b = _naive(pb)
    for i, (x, y) in enumerate(zip(res[:5], b[:5])):
        assert [int(v) for v in x] == y, (i, pb.what)
    assert res[5].tolist() == [list(r) for r in b[5]], pb.what
    _check_invariants(pb, res, oracle)
    if pb.matched:
        _check_flow(pb, res, oracle)
