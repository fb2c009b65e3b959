#!/usr/bin/env python
"""Multi-GPU parity check of the sharded place pods with reasons (run under torchrun on the GPUs of one box; not collected
by pytest).  One process per GPU, peer buffers mapped with IPC handles (dra_shard_export / dra_peer_import), so every state
word, packet and reasons slice crosses NVLink.  The call runs in the dense form and with 8 random candidates, under both
flags, each time from the pristine inventory (DRA_F_FRESH_INVENTORY).  Every rank's table, pod_node and own inventory
range must equal the CPU oracle's (tests/place_why_oracle.py), and so must every rank's four reason outputs.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_place_why_check.py
"""
import numpy as np
import torch

from multi_gpu_rank import dv, finish, join, pkg, report, start
import place_why_oracle as PW
R = pkg.records
F_EXH, F_FRESH = pkg.api.F_EXHAUSTIVE, pkg.api.F_FRESH_INVENTORY
WHY_N = pkg.api.WHY_N

rank, world, dev, stream = start()
w, pod_off = pkg.synth.pods(600, 12 * world, 23)
n_node, n_pod = w.n_node, len(pod_off) - 1
bounds = [n_node * r // world for r in range(world)] + [n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
join(ctx, bounds, world - 1, max(w.n_claim, 1), place=(n_pod,), why=(n_pod * n_node,))
keep = [dv(w.claims), dv(pod_off)]


def check(what, cn, co, flags):
    ref = PW.place_why(w.gpus, w.node_off, w.table, w.claims, pod_off, cn, co, None, len(w.claims), flags & F_EXH)
    n_pair = 0 if co is None else int(co[-1])
    n_why = n_pod * n_node if co is None else n_pair
    d_n = dv(cn) if cn is not None else None
    d_o = dv(co) if co is not None else None
    sizes = (n_pod * 4, n_why, n_why * 4, n_pod * WHY_N * 4, len(w.claims) * 4)
    outs = [torch.zeros(s + 16, dtype=torch.uint8, device=dev) for s in sizes]
    torch.cuda.synchronize()
    ctx.place_pods_why_global_device(keep[0].data_ptr(), len(w.claims), keep[1].data_ptr(), n_pod,
                                     d_n.data_ptr() if d_n is not None else None,
                                     d_o.data_ptr() if d_o is not None else None, n_pair, None, len(w.claims),
                                     *[o.data_ptr() for o in outs], flags=flags | F_FRESH)
    ctx.sync()
    table = ctx.gather_read(np.zeros(len(w.claims), dtype=R.OUT_DTYPE))
    got = [o.cpu().numpy()[:s].view(d) for o, s, d in zip(outs, sizes, (np.uint32, np.uint8, np.uint32, np.uint32, np.uint32))]
    inv = ctx.get_inventory()
    ok = table.tobytes() == ref[0].tobytes() and got[0].tobytes() == ref[1].tobytes() and \
        inv[g0:g1].tobytes() == ref[2][g0:g1].tobytes() and \
        all(x.tobytes() == np.ascontiguousarray(y, x.dtype).tobytes() for x, y in zip(got[1:], ref[3:]))
    report(f"sharded place pods with reasons, {what}", ok,
           f"{n_pod} pods, {int((ref[1] != 0xFFFFFFFF).sum())} placed, {n_why} pairs, {world} ranks")


rng = np.random.default_rng(5)
forms = {"dense": (None, None),
         "8 random": (rng.integers(0, n_node + 2, n_pod * 8).astype(np.uint32), (np.arange(n_pod + 1) * 8).astype(np.uint32))}
for name, (cn, co) in forms.items():
    for flags, fname in ((0, "first-fit"), (F_EXH, "exhaustive")):
        check(f"{name}, {fname}", cn, co, flags)
finish([ctx])
