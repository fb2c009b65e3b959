#!/usr/bin/env python
"""Multi-GPU parity check of the sharded preemption call (run under torchrun on the GPUs of one box; not collected by
pytest).  One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import), so every partial
crosses NVLink.  Each rank holds the real world on its own node range and the empty inventory elsewhere; the call runs in
the dense form and with 16 random candidates, under both flags.  Every rank's six outputs must equal the CPU oracle's on
the real world, and no rank's inventory may change.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_preempt_check.py
"""
import numpy as np
import torch

from multi_gpu_rank import dv, finish, join, pkg, report, start
import preempt_oracle as P
F_EXH = pkg.api.F_EXHAUSTIVE

rank, world, dev, stream = start()
w = pkg.synth.preempt(n_node=32 * world, gpus_per_node=8, n_pending=200, seed=23)
n_node = len(w.node_off) - 1
n_pod = len(w.pod_off) - 1
bounds = [n_node * r // world for r in range(world)] + [n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
mine = w.empty.copy()
mine[g0:g1] = w.gpus[g0:g1]
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(mine, w.node_off)
join(ctx, bounds, 0, max(len(w.run_claims), 1), preempt=(n_pod, n_pod * n_node, 16))
keep = [dv(x) for x in (w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio, w.run_out)]
run = pkg.api.RunningPods(keep[3].data_ptr(), len(w.run_claims), keep[4].data_ptr(), len(w.run_pod_off) - 1,
                          keep[5].data_ptr(), None, keep[6].data_ptr(), len(w.run_out))


def check(what, cn, co, flags):
    ref = P.preempt(w.gpus, w.node_off, w.table, w.claims, w.pod_off, w.prio, w.run_claims, w.run_pod_off, w.run_prio,
                    w.run_out, None, cn, co, 16, P.F_EXHAUSTIVE if flags & F_EXH else 0)
    n_pair = n_pod * n_node if co is None else int(co[-1])
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    sizes = (n_pair, n_pair * 4, n_pod * 4, n_pod, n_pod * 4, n_pod * 16 * 4)
    outs = [torch.zeros(s + 16, dtype=torch.uint8, device=dev) for s in sizes]
    torch.cuda.synchronize()
    ctx.preempt_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), keep[2].data_ptr(), n_pod,
                              d_n.data_ptr() if d_n is not None else None, d_o.data_ptr() if d_o is not None else None,
                              n_pair, run, *[o.data_ptr() for o in outs], 16, flags)
    ctx.sync()
    dt = (np.uint8, np.uint32, np.uint32, np.uint8, np.uint32, np.uint32)
    got = [o.cpu().numpy()[:s].view(d) for o, s, d in zip(outs, sizes, dt)]
    ok = all(x.tobytes() == y.tobytes() for x, y in zip(got, ref)) and ctx.get_inventory().tobytes() == mine.tobytes()
    report(f"sharded preemption, {what}", ok, f"{n_pod} pods, {int((ref[3] == P.EVICT).sum())} evicting, {world} ranks")


rng = np.random.default_rng(5)
forms = {"dense": (None, None),
         "16 random": (rng.integers(0, n_node + 2, n_pod * 16).astype(np.uint32), (np.arange(n_pod + 1) * 16).astype(np.uint32))}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
finish([ctx])
