#!/usr/bin/env python
"""Multi-GPU parity check of the sharded reasons of UnsuitableNodes (run under torchrun on the GPUs of one box; not
collected by pytest).  One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import), so
every slice crosses NVLink.  Each rank holds the real world on its own node range and the empty inventory elsewhere; the
call runs in the dense form and with 16 random candidates, under both flags.  Every rank's four outputs must equal the CPU
oracle's (tests/why_oracle.py) on the real world, and no rank's inventory may change.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_why_check.py
"""
import numpy as np
import torch

from multi_gpu_rank import dv, finish, join, pkg, report, start
import why_oracle as Y
F_EXH = pkg.api.F_EXHAUSTIVE

rank, world, dev, stream = start()
w = pkg.synth.preempt(n_node=16 * world, gpus_per_node=8, n_pending=100, seed=29)
n_node = len(w.node_off) - 1
n_pod = len(w.pod_off) - 1
bounds = [n_node * r // world for r in range(world)] + [n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
mine = w.empty.copy()
mine[g0:g1] = w.gpus[g0:g1]
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(mine, w.node_off)
join(ctx, bounds, 0, 64, why=(n_pod * n_node,))
keep = [dv(w.claims), dv(w.pod_off)]


def check(what, cn, co, flags):
    ref = Y.why(w.gpus, w.node_off, w.table, w.claims, w.pod_off, cn, co, Y.F_EXHAUSTIVE if flags & F_EXH else 0)
    n_pair = n_pod * n_node if co is None else int(co[-1])
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    sizes = (n_pair, n_pair * 4, n_pod * Y.WHY_N * 4, len(w.claims) * 4)
    outs = [torch.zeros(s + 16, dtype=torch.uint8, device=dev) for s in sizes]
    torch.cuda.synchronize()
    ctx.unsuitable_why_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n_pod,
                                     d_n.data_ptr() if d_n is not None else None,
                                     d_o.data_ptr() if d_o is not None else None, n_pair, *[o.data_ptr() for o in outs],
                                     flags=flags)
    ctx.sync()
    dt = (np.uint8, np.uint32, np.uint32, np.uint32)
    got = [o.cpu().numpy()[:s].view(d) for o, s, d in zip(outs, sizes, dt)]
    ok = all(x.tobytes() == np.ascontiguousarray(y, x.dtype).tobytes() for x, y in zip(got, ref)) and \
        ctx.get_inventory().tobytes() == mine.tobytes()
    report(f"sharded unsuitable reasons, {what}", ok,
           f"{n_pod} pods, {int((ref[0] == Y.ST_OK).sum())} of {n_pair} pairs OK, {world} ranks")


rng = np.random.default_rng(7)
forms = {"dense": (None, None),
         "16 random": (rng.integers(0, n_node + 2, n_pod * 16).astype(np.uint32), (np.arange(n_pod + 1) * 16).astype(np.uint32))}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
finish([ctx])
