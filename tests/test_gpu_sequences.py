"""GPU suite: long call sequences on one context per path, every step byte for byte against the sequence model.

A driver process keeps one context for thousands of calls and reuses its pinned buffers.  What such a process depends on
and a one-call test cannot see is the state kept between calls: the inventory a resident kernel hands from one batch to
the next, the graph a replay takes for a call of the same shape, the device copies of the claims that every batch
overwrites.  Each test here runs about 400 steps of tests/sequences.py (Allocate of changing size, content, flags and
out_off; Deallocate of earlier batches; UnsuitableNodes; pods Allocate; place pods; preemption with and without disruption
budgets and preempt and place, whose running pods are the records the sequence placed and still holds; pod capacity;
node-sorted batches; new selectors, tables and inventories; one calibration; one batch with an out_off outside n_out;
one refused call of each pod call) on one inventory, through:
  direct    the default context: the single-launch kernel reads and writes the pinned buffers itself
  nodirect  copy-engine transfers around the kernel chain
  nofused   the counting sort + pack chain
  graph     the host call captured once per shape and replayed
  resident  the single-launch kernel stays up and takes each eligible batch by doorbell
  device    Allocate on torch CUDA tensors (dra_allocate_batch_device), the rest of the calls as on the host
Buffers: one claims, one out_off and one output buffer per context, sized to the largest step.  Each step writes its batch
into the buffers' prefix, so the tail holds valid claims of earlier, larger batches; the output buffer is filled with a
sentinel before every step, and after it the slots below n_out must equal the model and the rest must hold the sentinel.
The pod calls go through the raw ABI on outputs sized for the call, filled with a sentinel and SLACK elements longer.
The inventory is compared every 50 steps, at the end and after every step that must not change it or that places pods.
A batch's records are kept as the library returned them for the Deallocate steps, masked where the library's own
evicted_by says preempt and place released them."""
import ctypes as C
import time

import numpy as np
import pytest

import sequences as S

pytestmark = pytest.mark.gpu

N_STEPS = 400
CHECK_EVERY = 50
SLACK = 16
SENT = 0xA5
PATHS = ["direct", "nodirect", "nofused", "graph", "resident", "device"]


def _flags(A, path):
    return {"direct": 0, "nodirect": A.CFG_NO_DIRECT, "nofused": A.CFG_NO_FUSED, "graph": A.CFG_USE_GRAPH | A.CFG_NO_DIRECT,
            "resident": A.CFG_RESIDENT, "device": 0}[path]


@pytest.fixture(scope="module")
def sequences_(oracle):
    """The three inventories, each with its sequence and the model's answers (computed once for every path)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = []
    for k, inv in enumerate(S.standard_inventories(sms)):
        steps = S.make_sequence(inv, N_STEPS, 100 + k)
        S.Model(inv, oracle).run(steps)
        kinds = [s.kind for s in steps]
        assert {s.kind for s in steps} == S.KINDS and all(kinds.count(kind) >= 8 for kind in S.POD_CALLS), (inv.name, kinds)
        out.append((inv, steps))
    return out


def _same(got, want, what):
    if got.tobytes() != want.tobytes():
        a, b = got.view(np.uint8).reshape(len(got), -1), want.view(np.uint8).reshape(len(want), -1)
        bad = np.nonzero((a != b).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} records differ, first at {bad[0]}: "
                             f"cuda={got[bad[0]]} model={want[bad[0]]}")


def _served(s):
    """Whether the resident kernel takes this step (dra_allocate_batch's eligibility for it)."""
    return (s.kind in ("alloc", "error") and not (s.flags & ~S.F_FRESH) and 1 <= len(s.claims) <= S.STAGED_CAP
            and s.n_out <= 2 * S.STAGED_CAP)


def _p(x):
    return None if x is None else x.ctypes.data_as(C.c_void_p)


def _arr(x, dtype):
    return None if x is None else np.ascontiguousarray(x, dtype=dtype)


def raw_pod_call(A, ctx, s, run):
    """dra_<call>_batch of pod-call step s (running pods `run` for the preemption calls) on outputs sized for the call,
    every byte SENT and SLACK elements longer than the call may write.  Returns (rc, outputs in the order of s.expect)."""
    R = A.R
    n_pod = len(s.pod_off) - 1
    n_pair = n_pod * ctx.n_node if s.cand_off is None else int(s.cand_off[-1])
    u8, u16, u32, u64 = np.uint8, np.uint16, np.uint32, np.uint64
    pre = [(n_pair, u8), (n_pair, u32), (n_pod, u32), (n_pod, u8), (n_pod, u32), (n_pod * (s.arg or 0), u32)]
    sizes = {"place": [(s.n_out, R.OUT_DTYPE), (n_pod, u32)],
             "capacity": [(n_pair, u16), (n_pair, u8), (n_pod, u64), (n_pod, u32)],
             "preempt": pre, "preempt_pdb": pre + [(n_pair, u32), (n_pod, u32)],
             "preempt_place": [(s.n_out, R.OUT_DTYPE), (n_pod, u32), (n_pod, u8), (len(run.prio) if run else 0, u32)]}
    outs = [np.full((max(n, 1) + SLACK) * np.dtype(dt).itemsize, SENT, np.uint8).view(dt) for n, dt in sizes[s.base]]
    o = [_p(x) for x in outs]
    c, po, pr = _arr(s.claims, R.CLAIM_DTYPE), _arr(s.pod_off, u32), _arr(s.prio, np.int32)
    cn, co, oo = _arr(s.cand_nodes, u32), _arr(s.cand_off, u32), _arr(s.out_off, u32)
    L, h = ctx._lib, ctx._h
    if s.base == "place":
        return L.dra_place_pods_batch(h, _p(c), len(c), _p(po), n_pod, _p(cn), _p(co), _p(oo), o[0], s.n_out, o[1],
                                      s.flags), outs
    if s.base == "capacity":
        return L.dra_pod_capacity_batch(h, _p(c), len(c), _p(po), n_pod, _p(cn), _p(co), s.arg, *o, s.flags), outs
    keep = [_arr(run.claims, R.CLAIM_DTYPE), _arr(run.pod_off, u32), _arr(run.prio, np.int32), _arr(run.out, R.OUT_DTYPE),
            _arr(run.out_off, u32)]
    rc_, rpo, rpr, ro, roo = keep
    rp = A.RunningPods(rc_.ctypes.data, len(rc_), rpo.ctypes.data, len(rpo) - 1, rpr.ctypes.data, roo.ctypes.data,
                       ro.ctypes.data, len(ro))
    mv = s.arg
    if s.base == "preempt":
        rc = L.dra_preempt_batch(h, _p(c), len(c), _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(rp), *o[:5],
                                 o[5] if mv else None, mv, s.flags)
    elif s.base == "preempt_pdb":
        pdb = np.append(run.budgets(len(s.pdb_allowed)), np.uint32(S.NONE))     # (never empty: NULL means no array)
        al = _arr(s.pdb_allowed, np.int32)
        bud = A.DisruptionBudgets(pdb.ctypes.data, al.ctypes.data, len(al))
        rc = L.dra_preempt_pdb_batch(h, _p(c), len(c), _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(rp), C.byref(bud),
                                     o[0], o[1], o[6], o[2], o[3], o[4], o[7], o[5] if mv else None, mv, s.flags)
    else:
        rc = L.dra_preempt_place_batch(h, _p(c), len(c), _p(po), _p(pr), n_pod, _p(cn), _p(co), C.byref(rp), _p(oo),
                                       o[0], s.n_out, o[1], o[2], o[3], s.flags)
    return rc, outs


class Runner:
    def __init__(self, pkg, path, inv, steps):
        A, R = pkg.api, pkg.records
        self.A, self.path, self.inv, self.steps = A, path, inv, steps
        self.ctx = A.Context(device=0, flags=_flags(A, path))
        self.ctx.set_table(inv.tables[0])
        self.ctx.set_inventory(inv.gpus, inv.node_off)
        n_c = max(len(s.claims) for s in steps if s.claims is not None)
        n_o = max(s.n_out for s in steps) + 64
        self.pc = A.PinnedBuffer(n_c, R.CLAIM_DTYPE)
        self.pf = A.PinnedBuffer(n_c, np.uint32)
        self.po = A.PinnedBuffer(n_o, R.OUT_DTYPE)
        self.pc.array[:] = inv.pool[:n_c]                 # valid claims everywhere before the first batch
        self.pf.array[:] = np.arange(n_c, dtype=np.uint32)
        self.got = {}
        if path == "device":
            import torch
            self.torch = torch
            self.dc = torch.zeros(n_c * 16, dtype=torch.uint8, device="cuda")
            self.df = torch.zeros(n_c, dtype=torch.int32, device="cuda")
            self.do = torch.zeros(n_o, dtype=torch.int64, device="cuda")
            self.dc.copy_(torch.from_numpy(self.pc.array.view(np.uint8).copy()))
            torch.cuda.synchronize()

    def close(self):
        self.ctx.close()
        for p in (self.pc, self.pf, self.po):
            p.free()

    def allocate(self, s):
        """One Allocate step through this context's path; returns the whole output buffer after it."""
        c, n = self.ctx, len(s.claims)
        self.pc.array[:n] = s.claims
        if s.out_off is not None:
            self.pf.array[:n] = s.out_off
        self.po.array[:] = S.SENTINEL
        if self.path != "device":
            c.allocate(self.pc.array[:n], None if s.out_off is None else self.pf.array[:n], s.n_out, flags=s.flags,
                       out=self.po.array)
            return self.po.array
        torch = self.torch
        self.dc[: n * 16].copy_(torch.from_numpy(self.pc.array[:n].view(np.uint8).copy()))
        if s.out_off is not None:
            self.df[:n].copy_(torch.from_numpy(self.pf.array[:n].view(np.int32).copy()))
        self.do.fill_(int(self.po.array[:1].view(np.int64)[0]))
        torch.cuda.synchronize()                          # (the context's stream does not wait for torch's)
        try:
            c.allocate_device(self.dc.data_ptr(), n, None if s.out_off is None else self.df.data_ptr(),
                              self.do.data_ptr(), s.n_out, s.flags)
            c.sync()
        finally:
            self.po.array[:] = self.do.cpu().numpy().view(self.po.array.dtype)
        return self.po.array

    def run(self):
        A, c, inv, steps = self.A, self.ctx, self.inv, self.steps
        served = replays = 0
        b0 = c.serve_batches()
        prev_chain = None
        for i, s in enumerate(steps):
            what = f"{self.path} {inv.name} step {i} ({s.kind})"
            if s.kind in ("alloc", "sorted", "error", "sorted_bad"):
                l0 = c.launch_count()
                if s.kind in ("error", "sorted_bad"):
                    with pytest.raises(A.DraError) as e:
                        self.allocate(s)
                    assert e.value.code == A.E_INVAL, what
                    out = self.po.array
                else:
                    out = self.allocate(s)
                    _same(out[: s.n_out], s.expect, what)
                    self.got[i] = S.held(s, out[: s.n_out], None, 0, inv.node_off)
                tail = out[s.n_out:]
                assert tail.tobytes() == S.SENTINEL.tobytes() * len(tail), f"{what}: a write past n_out"
                chain = c.last_chain()
                if self.path == "resident":
                    if _served(s):
                        served += 1
                        assert chain == {"serve"}, f"{what}: took {sorted(chain)}"
                    else:
                        assert "serve" not in chain, what
                if self.path == "graph" and s.kind == "alloc":
                    assert "fused_direct" not in chain and "serve" not in chain, what
                    assert c.launch_count() - l0 == len(chain), f"{what}: {c.launch_count() - l0} launches for {sorted(chain)}"
                    if i >= 2 and s.key() == steps[i - 1].key() == steps[i - 2].key():
                        replays += 1
                        assert chain == prev_chain, what
                    prev_chain = chain
                if s.kind == "sorted_bad":
                    assert c.get_inventory().tobytes() == s.live_after.tobytes(), f"{what}: the inventory changed"
            elif s.kind == "dealloc":
                for b in s.batches:
                    h = self.got.pop(b)
                    c.deallocate(h.claims, h.out, h.out_off)
            elif s.kind == "unsuitable":
                bits = c.unsuitable(s.claims, s.pod_off, s.cand_nodes, s.cand_off, s.flags)
                assert bits.tobytes() == s.expect.tobytes(), what
                assert c.get_inventory().tobytes() == s.live_after.tobytes(), f"{what}: the inventory changed"
            elif s.kind == "pods":
                out = c.allocate_pods(s.claims, s.pod_off, s.out_off, s.n_out, s.flags)
                _same(out, s.expect, what)
                self.got[i] = S.held(s, out, None, 0, inv.node_off)
            elif s.base in S.POD_CALLS:
                self.pod_call(i, s, what)
            elif s.kind == "selectors":
                c.set_gpu_attrs(inv.attrs if s.arg else None)
                c.set_selectors(inv.sels if s.arg else None)
            elif s.kind == "table":
                c.set_table(inv.tables[s.arg])
            elif s.kind == "reset":
                c.reset_inventory()
            elif s.kind == "set_inventory":
                c.set_inventory(s.live_after, inv.node_off)
            elif s.kind == "calibrate":
                c.calibrate()
            elif s.kind == "idle" and self.path == "resident":
                time.sleep(0.05)                          # longer than the resident kernel's 20 ms idle time-out
            elif s.kind == "restart" and self.path == "resident":
                c.serve_stop()
                c.serve_start()
            if i % CHECK_EVERY == CHECK_EVERY - 1 or i == len(steps) - 1:
                _same(c.get_inventory(), s.live_after, f"{what}: inventory")
        if self.path == "resident":
            assert served >= 100 and c.serve_batches() - b0 == served, (served, c.serve_batches() - b0)
        if self.path == "graph":
            assert replays >= 10, replays
        return served, replays

    def pod_call(self, i, s, what):
        """one place, capacity or preemption step: outputs, slack and inventory against the model; the records it places
        kept for Deallocate, and the running pods it evicts masked in theirs"""
        A, c, inv = self.A, self.ctx, self.inv
        run = None
        if s.base in S.PREEMPT_KINDS:
            run = S.running(s.batches, [self.got[b] for b in s.batches])
            if s.kind in ("preempt_bad", "preempt_pdb_bad"):
                run = S.two_node_pod(run, inv.gpus, inv.node_off)
        rc, outs = raw_pod_call(A, c, s, run)
        if s.expect is None:
            assert rc == A.E_INVAL, f"{what}: rc {rc}"
            assert all((o.view(np.uint8) == SENT).all() for o in outs), f"{what}: an output was written"
        else:
            assert rc == A.OK, f"{what}: rc {rc}"
            for k, (o, y) in enumerate(zip(outs, s.expect)):
                _same(o[: y.size], y.reshape(-1), f"{what}: output {k}")
                assert (o[y.size:].view(np.uint8) == SENT).all(), f"{what}: written past output {k}"
            n_pod = len(s.pod_off) - 1
            if s.base == "preempt_place":
                S.release(self.got, run, outs[3][: len(run.prio)], inv.n_node)
            if s.base in ("place", "preempt_place"):
                self.got[i] = S.held(s, outs[0][: s.n_out], outs[1][:n_pod], 0, inv.node_off)
            assert "serve" not in c.last_chain(), f"{what}: took {sorted(c.last_chain())}"
        _same(c.get_inventory(), s.live_after, f"{what}: inventory")


@pytest.mark.parametrize("inv_ix", [0, 1, 2], ids=["sms_minus_1_nodes", "mixed_60_nodes", "mig16_48_nodes"])
@pytest.mark.parametrize("path", PATHS)
def test_long_sequence_matches_model(pkg, sequences_, request, path, inv_ix):
    inv, steps = sequences_[inv_ix]
    r = Runner(pkg, path, inv, steps)
    request.addfinalizer(r.close)        # (after the failure report, which shows arrays that live in the pinned buffers)
    r.run()
