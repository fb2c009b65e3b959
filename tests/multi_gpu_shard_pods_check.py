#!/usr/bin/env python
"""Multi-GPU parity check of the sharded pods Allocate (run under torchrun on the GPUs of one box; not collected by
pytest).  One process per GPU, gather buffers mapped with IPC handles (dra_shard_export / dra_peer_import).  The classic
flow on a sharded world: a sharded Allocate without DRA_F_FRESH_INVENTORY makes the ranks' inventories diverge, a sharded
exhaustive UnsuitableNodes finds a suitable node for each pod, and the sharded pods Allocate places the pods retargeted to
those nodes.  Every rank's verdict, whole table and own inventory range must equal the CPU oracle's on the real state.
Then the same pods call with first-fit, exhaustive and fresh-inventory flags on the fragmented pod workload.

  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/multi_gpu_shard_pods_check.py
"""
import importlib, os, sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("k8s-dra-driver_b200")
from oracle import oracle as O
R = pkg.records
F_EXH, F_FRESH = pkg.api.F_EXHAUSTIVE, pkg.api.F_FRESH_INVENTORY

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
os.environ.setdefault("NCCL_DEBUG", "WARN")
torch.cuda.set_device(local)
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
dev = torch.device("cuda", local)
stream = torch.cuda.Stream(device=dev); torch.cuda.set_stream(stream)
fails = 0

w, pod_off = pkg.synth.pods(2000, 24 * world, 11)
bounds = [w.n_node * r // world for r in range(world)] + [w.n_node]
g0, g1 = int(w.node_off[bounds[rank]]), int(w.node_off[bounds[rank + 1]])
first = int(pod_off[300])                           # the first 300 pods' claims: the sharded claim Allocate
n_pod = 1700
claims = w.claims[first:].copy()
po = (pod_off[300:] - first).astype(np.uint32)
ctx = pkg.api.Context(device=local, stream=stream.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
uid = [pkg.api.Context.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
ctx.comm_init(uid[0], rank, world)
ctx.set_shard_map(bounds, stray_rank=world - 1)
ctx.set_shard_pairs(n_pod * w.n_node)
hs = [None] * world
dist.all_gather_object(hs, ctx.shard_export(max(w.n_claim, 1)))
ctx.peer_import(hs)


def dv(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev)


def real_state():
    """Every rank's inventory over its own GPU range, assembled on every rank."""
    mine = ctx.get_inventory()
    parts = [None] * world
    dist.all_gather_object(parts, mine[g0:g1].tobytes())
    real = w.gpus.copy()
    for r in range(world):
        a, b = int(w.node_off[bounds[r]]), int(w.node_off[bounds[r + 1]])
        real[a:b] = np.frombuffer(parts[r], dtype=w.gpus.dtype)
    return real


def check(what, c, p_off, flags):
    global fails
    src = w.gpus if flags & F_FRESH else real_state()
    ref, ref_inv = O.allocate_pods(src, w.node_off, w.table, c, p_off, None, len(c), O.F_EXHAUSTIVE if flags & F_EXH else 0)
    d_c, d_p = dv(c), dv(p_off)
    torch.cuda.synchronize()
    ctx.allocate_pods_global_device(d_c.data_ptr(), len(c), d_p.data_ptr(), len(p_off) - 1, None, len(c), flags)
    ctx.sync()
    got = ctx.gather_read(np.zeros(len(c), dtype=R.OUT_DTYPE))
    inv = ctx.get_inventory()
    ok = got.tobytes() == ref.tobytes() and inv[g0:g1].tobytes() == ref_inv[g0:g1].tobytes()
    t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
    fails += int(t.item()) != 0
    if rank == 0:
        st = ref["status"]
        print(f"sharded pods Allocate, {what}: {'OK' if int(t.item()) == 0 else 'MISMATCH'} "
              f"({len(p_off) - 1} pods, {int((st == 0).sum())} OK slots of {len(st)}, {world} ranks)")
    return ref


# 1. sharded claim Allocate: the ranks' copies diverge outside their ranges
d_first = dv(w.claims[:first])
ctx.allocate_global_device(d_first.data_ptr(), first, None, first, 0)
ctx.gather_read(np.zeros(first, dtype=R.OUT_DTYPE))
# 2. sharded exhaustive UnsuitableNodes on the real state
n_pair = n_pod * w.n_node
d_c, d_p = dv(claims), dv(po)
bits = torch.zeros((n_pair + 7) // 8, dtype=torch.uint8, device=dev)
ctx.unsuitable_global_device(d_c.data_ptr(), len(claims), d_p.data_ptr(), n_pod, None, None, n_pair, bits.data_ptr(), F_EXH)
ctx.sync()
real = real_state()
dn = np.tile(np.arange(w.n_node, dtype=np.uint32), n_pod)
do = (np.arange(n_pod + 1, dtype=np.uint64) * w.n_node).astype(np.uint32)
ref_bits = O.unsuitable(real, w.node_off, w.table, claims, po, dn, do, flags=O.F_EXHAUSTIVE)
h = bits.cpu().numpy()
ok = h.tobytes() == ref_bits.tobytes()
t = torch.tensor([0 if ok else 1], device=dev); dist.all_reduce(t)
fails += int(t.item()) != 0
if rank == 0:
    print(f"sharded exhaustive UnsuitableNodes: {'OK' if int(t.item()) == 0 else 'MISMATCH'} ({n_pair} pairs)")
# 3. one suitable node per pod (at most one pod per node), claims retargeted there: every pod must be placed
verdict = np.unpackbits(h, bitorder="little")[:n_pair].reshape(n_pod, w.n_node)
taken, keep = set(), []
for p in range(n_pod):
    free = [n for n in np.flatnonzero(verdict[p]) if n not in taken]
    if free:
        n = int(free[0]); taken.add(n); keep.append((p, n))
sub = np.concatenate([claims[po[p]: po[p + 1]] for p, _ in keep]).copy()
sub_off = np.zeros(len(keep) + 1, dtype=np.uint32)
sub_off[1:] = np.cumsum([po[p + 1] - po[p] for p, _ in keep])
for k, (_, n) in enumerate(keep):
    sub["node"][sub_off[k]: sub_off[k + 1]] = n
ref = check("pods on their suitable nodes, exhaustive", sub, sub_off, F_EXH)
if not (ref["status"] == 0).all():
    fails += 1
    if rank == 0:
        print("MISMATCH: a pod the exhaustive verdict called suitable was not placed")
# 4. the fragmented workload itself, every flag; repeated calls use both table parities
for flags, name in ((0, "first-fit"), (F_EXH, "exhaustive"), (F_FRESH, "fresh first-fit"), (F_EXH | F_FRESH, "fresh exhaustive")):
    check(name, claims, po, flags)
dist.barrier()
ctx.close()
t = torch.tensor([fails], device=dev); dist.all_reduce(t)
if rank == 0:
    print("ALL OK" if int(t.item()) == 0 else f"{int(t.item())} FAILURES")
dist.destroy_process_group()
sys.exit(1 if int(t.item()) else 0)
