"""Per-CTA phase timeline of k_fused on the cfg2 batch (instrumentation: DRA_TIMELINE=1).
  DRA_TIMELINE=1 python profiles/timeline.py   (on a GPU box)"""
import importlib, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
pkg = importlib.import_module("k8s-dra-driver_b200")
w = pkg.synth.cfg2()
s = torch.cuda.Stream(); torch.cuda.set_stream(s)
ctx = pkg.api.Context(device=0, stream=s.cuda_stream)
ctx.set_table(w.table); ctx.set_inventory(w.gpus, w.node_off)
d_claims = torch.from_numpy(w.claims.view(np.uint8).copy()).cuda()
d_out = torch.zeros(w.n_out * 8, dtype=torch.uint8, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for it in range(6):
    flush.fill_(1)
    ctx.allocate_device(d_claims.data_ptr(), w.n_claim, None, d_out.data_ptr(), w.n_out, pkg.api.F_FRESH_INVENTORY)
    ctx.sync()
tl = ctx.debug_timeline(w.n_node + 1).astype(np.uint64)
node = tl[: w.n_node]
names = ["entry: table/inventory copies issued", "filter", "sync", "table/inventory wait + first fetch", "pack (warp 0)"]
for k, nm in enumerate(names):
    d = (node[:, k + 2] - node[:, k + 1]).astype(np.int64)
    print(f"{nm:36s} cycles: median {int(np.median(d)):6d}  p90 {int(np.percentile(d, 90)):6d}  max {int(d.max()):6d}")
tot = (node[:, 6] - node[:, 1]).astype(np.int64)
cnt = (node[:, 7] & np.uint64(0xFFFF)).astype(np.int64); nlive = ((node[:, 7] >> np.uint64(16)) & np.uint64(0xFFFF)).astype(np.int64)
fetch = ((node[:, 7] >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.int64); pre_a = (node[:, 7] >> np.uint64(48)).astype(np.int64)
pre = (node[:, 0] & np.uint64(0xFFFFF)).astype(np.int64); loop = ((node[:, 0] >> np.uint64(20)) & np.uint64(0xFFFFF)).astype(np.int64); epi = (node[:, 0] >> np.uint64(40)).astype(np.int64)
print("total in-CTA cycles: median %d  max %d" % (np.median(tot), tot.max()))
print("claims/node median %d max %d; live records/node median %d max %d" % (np.median(cnt), cnt.max(), np.median(nlive), nlive.max()))
print("inside pack: pre-pass median %d  serial loop median %d (%.0f cycles/live record)  epilogue median %d" % (np.median(pre), np.median(loop), np.median(loop / np.maximum(nlive, 1)), np.median(epi)))
print("  pre-pass part a (validity/range/dead-shape emission) median %d; next-segment fetch median %d; pack minus (pre+loop+epi+fetch) median %d" % (np.median(pre_a), np.median(fetch), np.median((node[:, 6] - node[:, 5]).astype(np.int64) - pre - loop - epi - fetch)))
i = int(np.argmax(tot)); print("slowest CTA", i, "pack", int(node[i, 6] - node[i, 5]), "pre/loop/epi", int(pre[i]), int(loop[i]), int(epi[i]), "claims", int(cnt[i]), "live", int(nlive[i]))

# ---- direct host I/O (the host call): phases of CTA 0 in wall-clock ns (globaltimer) ----
pin_c = pkg.api.PinnedBuffer(w.n_claim, pkg.records.CLAIM_DTYPE); pin_c.array[:] = w.claims
pin_o = pkg.api.PinnedBuffer(w.n_out, pkg.records.OUT_DTYPE)
import time
for it in range(6):
    flush.fill_(1); torch.cuda.synchronize()
    t0 = time.perf_counter()
    ctx.allocate_raw(pin_c.ptr, w.n_claim, None, pin_o.ptr, w.n_out, pkg.api.F_FRESH_INVENTORY)
    dt = time.perf_counter() - t0
tl = ctx.debug_timeline(w.n_node + 3).astype(np.uint64)
d = tl[w.n_node + 2].astype(np.int64)
if d[0]:
    print("direct host I/O, CTA 0 (ns): ingest loads+stores %d | barrier 1 %d | body %d | barrier 2 (wait for the slowest CTA) %d | egress %d | total %d ; host call %.1f us"
          % (d[1] - d[0], d[2] - d[1], d[3] - d[2], d[4] - d[3], d[5] - d[4], d[5] - d[0], dt * 1e6))
