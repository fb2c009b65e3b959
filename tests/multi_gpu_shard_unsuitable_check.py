#!/usr/bin/env python
"""Multi-GPU parity check of sharded UnsuitableNodes (run under torchrun on N >= 2 GPUs of one box; not collected by
pytest).  One process per GPU, gather buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  A sharded
Allocate without DRA_F_FRESH_INVENTORY first makes the ranks' inventories diverge; then every rank's whole bitmap from
dra_unsuitable_batch_global_device must equal the CPU oracle's answer on the state that Allocate left — dense and
candidate-list forms, first-fit and exhaustive, claims of every kind with counts > 1 and malformed claims.

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/multi_gpu_shard_unsuitable_check.py
"""
import numpy as np
import torch

from multi_gpu_rank import dv, finish, join, pkg, report, start
from oracle import oracle as O
R = pkg.records

rank, world, dev, stream = start()
w = pkg.synth.mixed(9000, 97, 41)
ranges = pkg.shard.plan(w.claims["node"], w.n_node, world)
n_pod = 800
pods = w.claims[:n_pod].copy()
pod_off = np.arange(n_pod + 1, dtype=np.uint32)
rng = np.random.default_rng(7)
per = rng.integers(0, 12, n_pod)
cand_off = np.zeros(n_pod + 1, dtype=np.uint32); cand_off[1:] = np.cumsum(per)
cand_nodes = rng.integers(0, w.n_node + 3, int(cand_off[-1])).astype(np.uint32)      # some name no node
ctx = pkg.api.Context(device=dev.index, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
join(ctx, [r[0] for r in ranges] + [ranges[-1][1]], 0, w.n_out, pairs=(n_pod * w.n_node,))

d_claims, d_off = dv(w.claims), dv(w.out_off)
ctx.allocate_global_device(d_claims.data_ptr(), w.n_claim, d_off.data_ptr(), w.n_out, 0)
ctx.gather_read(np.zeros(w.n_out, dtype=R.OUT_DTYPE))
_, real = O.allocate(w.gpus, w.node_off, w.table, w.claims, w.out_off, w.n_out)
d_pods, d_po, d_cn, d_co = dv(pods), dv(pod_off), dv(cand_nodes), dv(cand_off)
dense_cn = np.tile(np.arange(w.n_node, dtype=np.uint32), n_pod)
dense_co = (np.arange(n_pod + 1, dtype=np.uint64) * w.n_node).astype(np.uint32)
for rep in range(2):                                   # repeated calls: both staging parities, rising sequence numbers
    for flags, oflags in ((0, 0), (pkg.api.F_EXHAUSTIVE, O.F_EXHAUSTIVE)):
        for form, cn, co, dcn, dco in (("dense", dense_cn, dense_co, None, None), ("candidates", cand_nodes, cand_off, d_cn, d_co)):
            n_pair = int(co[-1])
            bits = torch.zeros((n_pair + 7) // 8, dtype=torch.uint8, device=dev)
            ctx.unsuitable_global_device(d_pods.data_ptr(), n_pod, d_po.data_ptr(), n_pod, None if dcn is None else dcn.data_ptr(),
                                         None if dco is None else dco.data_ptr(), n_pair, bits.data_ptr(), flags)
            ctx.sync()
            ref = O.unsuitable(real, w.node_off, w.table, pods, pod_off, cn, co, flags=oflags)
            report(f"sharded UnsuitableNodes rep {rep}, {form}, flags {flags}", bits.cpu().numpy().tobytes() == ref.tobytes(),
                   f"{n_pair} pairs, {world} ranks")
finish([ctx])
