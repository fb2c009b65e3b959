#!/usr/bin/env python
"""Multi-GPU parity check of the sharded place pods (run under torchrun on the GPUs of one box; not collected by pytest).
One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import), so every state word and
packet crosses NVLink.  A sharded Allocate without DRA_F_FRESH_INVENTORY first makes the ranks' inventories diverge; then
the place-pods call runs in the dense form, with 8 random candidates and with every node descending, under every flag.
Every rank's whole table, pod_node and own inventory range must equal the CPU oracle's on the real state.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_place_check.py
"""
import numpy as np
import torch
import torch.distributed as dist

from multi_gpu_rank import dv, finish, join, pkg, report, start
import place_oracle as P
R = pkg.records
F_EXH, F_FRESH = pkg.api.F_EXHAUSTIVE, pkg.api.F_FRESH_INVENTORY

rank, world, dev, stream = start()
w, pod_off = pkg.synth.pods(2000, 24 * world, 17)
bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
first = int(pod_off[300])
claims = w.claims[first:].copy()
po = (pod_off[300:] - first).astype(np.uint32)
n_pod = len(po) - 1
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
join(ctx, bounds, world - 1, max(w.n_claim, 1), place=(n_pod,))


def real_state():
    parts = [None] * world
    dist.all_gather_object(parts, ctx.get_inventory()[g0:g1].tobytes())
    real = w.gpus.copy()
    for r in range(world):
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        real[a:b] = np.frombuffer(parts[r], dtype=w.gpus.dtype)
    return real


def check(what, cn, co, flags):
    src = w.gpus if flags & F_FRESH else real_state()
    ref, ref_node, ref_inv = P.place_pods(src, w.node_off, w.table, claims, po, cn, co, None, len(claims),
                                          P.F_EXHAUSTIVE if flags & F_EXH else 0)
    d_c, d_p = dv(claims), dv(po)
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    d_pn = torch.zeros(n_pod * 4, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    ctx.place_pods_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n_pod, d_n.data_ptr() if d_n is not None else None,
                                 d_o.data_ptr() if d_o is not None else None, int(co[-1]) if co is not None else 0, None,
                                 len(claims), d_pn.data_ptr(), flags)
    ctx.sync()
    got = ctx.gather_read(np.zeros(len(claims), dtype=R.OUT_DTYPE))
    node = d_pn.cpu().numpy().view(np.uint32)
    inv = ctx.get_inventory()
    ok = got.tobytes() == ref.tobytes() and node.tobytes() == ref_node.tobytes() and inv[g0:g1].tobytes() == ref_inv[g0:g1].tobytes()
    report(f"sharded place pods, {what}", ok, f"{n_pod} pods, {int((ref_node != 0xFFFFFFFF).sum())} placed, {world} ranks")


d_first = dv(w.claims[:first])
ctx.allocate_global_device(d_first.data_ptr(), first, None, first, 0)
ctx.gather_read(np.zeros(first, dtype=R.OUT_DTYPE))
rng = np.random.default_rng(5)
asc = np.tile(np.arange(w.n_node, dtype=np.uint32), n_pod)
every = (np.arange(n_pod + 1) * w.n_node).astype(np.uint32)
forms = {"dense": (None, None),
         "8 random": (rng.integers(0, w.n_node + 2, n_pod * 8).astype(np.uint32), (np.arange(n_pod + 1) * 8).astype(np.uint32)),
         "descending": (asc[::-1].copy(), every)}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive"), (F_FRESH, "fresh first-fit"), (F_EXH | F_FRESH, "fresh exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
finish([ctx])
