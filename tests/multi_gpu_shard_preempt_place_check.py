#!/usr/bin/env python
"""Multi-GPU check of the sharded preempt-and-place call (run under torchrun on the GPUs of one box; not collected by
pytest).  One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import), so the state
exchange and the verdict agreement cross NVLink between processes.  Each rank holds the real world on its own node range
and the empty inventory elsewhere; the call runs in the dense form and with 16 random candidates, under both flags, each
call from the world as loaded.  Every rank's table, pod_node, pod_status and evicted_by must equal the CPU oracle's on the
real world, its own range must equal the oracle's final inventory, and the rest of its copy must be unchanged.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_preempt_place_check.py
"""
import numpy as np
import torch

from multi_gpu_rank import dv, finish, join, pkg, report, start
import preempt_place_oracle as PP
R = pkg.records
F_EXH = pkg.api.F_EXHAUSTIVE

rank, world, dev, stream = start()
w = pkg.synth.preempt(n_node=32 * world, gpus_per_node=8, n_pending=200, seed=29)
n_node = len(w.node_off) - 1
n_pod = len(w.pod_off) - 1
n_run = len(w.run_pod_off) - 1
bounds = [n_node * r // world for r in range(world)] + [n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
mine = w.empty.copy()
mine[g0:g1] = w.gpus[g0:g1]
placed = w.claims.copy(); placed["node"] = 0
sl = R.claim_slots(placed, 1).astype(np.int64)
out_off = np.concatenate([[0], np.cumsum(sl)[:-1]]).astype(np.uint32)
n_out = int(sl.sum())
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(mine, w.node_off)
join(ctx, bounds, 0, n_out, preempt_place=(n_pod, n_pod * n_node, n_run))
keep = [dv(x) for x in (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out, out_off)]
run = pkg.api.RunningPods(keep[3].data_ptr(), len(w.run_claims), keep[4].data_ptr(), n_run,
                          keep[5].data_ptr(), None, keep[6].data_ptr(), len(w.run_out))


def check(what, cn, co, flags):
    ref = PP.preempt_place(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off,
                           w.run_prio, w.run_out, None, cn, co, out_off, n_out, PP.F_EXHAUSTIVE if flags & F_EXH else 0)
    ctx.set_inventory(mine, w.node_off)                        # every call from the world as loaded
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    outs = [torch.zeros(s, dtype=torch.uint8, device=dev) for s in (n_pod * 4, n_pod, n_run * 4)]
    torch.cuda.synchronize()
    ctx.preempt_place_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                                    d_n.data_ptr() if d_n is not None else None, d_o.data_ptr() if d_o is not None else None,
                                    0 if co is None else int(co[-1]), run, keep[7].data_ptr(), n_out,
                                    *[o.data_ptr() for o in outs], flags)
    ctx.sync()
    table = ctx.gather_read(np.zeros(n_out, dtype=R.OUT_DTYPE))
    got = [table] + [o.cpu().numpy().view(d) for o, d in zip(outs, (np.uint32, np.uint8, np.uint32))]
    inv = ctx.get_inventory()
    ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref[:4]))
    ok = ok and inv[g0:g1].tobytes() == ref[4][g0:g1].tobytes()
    ok = ok and inv[:g0].tobytes() == mine[:g0].tobytes() and inv[g1:].tobytes() == mine[g1:].tobytes()
    report(f"sharded preempt and place, {what}", ok, f"{n_pod} pods, {int((ref[2] == PP.EVICT).sum())} evicting, {world} ranks")


rng = np.random.default_rng(5)
forms = {"dense": (None, None),
         "16 random": (rng.integers(0, n_node + 2, n_pod * 16).astype(np.uint32), (np.arange(n_pod + 1) * 16).astype(np.uint32))}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
finish([ctx])
