/*
 * dra_alloc.h — C ABI of libdra_alloc.so, the H100 (sm_90a) allocation hot path.
 *
 * This is the drop-in boundary for ONE path of NVIDIA/k8s-dra-driver: the per-node GPU/MIG claim search
 * behind the classic-DRA controller surface  Allocate() / UnsuitableNodes() / Deallocate()  that
 * BASELINE.json's north_star names.  That surface is ABSENT from the reference snapshot
 * (cmd/nvidia-dra-controller/ holds only main.go, imex.go, types.go — SURVEY.md F1); each entry point
 * below cites the reference interface it stands in for or the reference code that fixes its semantics.
 * A Go driver binds these with cgo (INTEGRATION.md shows the stub); tests bind them with ctypes.
 *
 * Plain C: pointers + sizes, caller-owned buffers, int return codes, no callbacks, no torch types.
 * Semantics are normative in spec/ALLOCATION.md; oracle/ is the CPU checker, never linked here.
 *
 * Threading: one in-flight call per dra_ctx (the reference serialises the same way with a global mutex,
 * cmd/nvidia-dra-plugin/driver.go:119-120, device_state.go:129-130).  Distinct contexts are independent.
 */
#ifndef DRA_ALLOC_H
#define DRA_ALLOC_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DRA_ABI_VERSION      2u   /* 2: flags on dra_unsuitable_batch, pod mode, sharded global batch, resident mode */

#define DRA_MAX_GPUS_PER_NODE 32u   /* one warp lane per GPU of a node */
#define DRA_MAX_MODELS        16u
#define DRA_MAX_PROFILES      16u   /* NVML GPU_INSTANCE_PROFILE_COUNT is 10 (go-nvml const.go:764-765) */
#define DRA_MAX_COUNT         32u   /* devices per GPU claim; k8s caps results per claim at 32
                                       (vendor/k8s.io/api/resource/v1beta1/types.go:792) */
#define DRA_MAX_GROUP         32u   /* members of one co-location run (same cap) */
#define DRA_MAX_POD           32u   /* claims of one pod in pod mode (spec §12) */
#define DRA_EXH_BUDGET        4096u /* descents of the exhaustive placement search per pod evaluation (spec §12) */
#define DRA_GPU_NONE          0xFFFFFFFFu

/* ---- records (spec/ALLOCATION.md §1) ------------------------------------------------------------ */

/* One physical GPU.  Mirrors the fields of GpuInfo that matter to allocation
 * (cmd/nvidia-dra-plugin/deviceinfo.go:30-43: index, migEnabled, memoryBytes) plus the occupancy the
 * removed NodeAllocationState CRD carried.  busy bit i = memory slice i in use
 * (deviceinfo.go:199-204, go-nvml nvml.h:9761-9765). */
typedef struct dra_gpu_rec {
    uint16_t busy;
    uint8_t  flags;         /* DRA_GPU_* */
    uint8_t  model;         /* row of the placement table */
    uint32_t mem_free_mib;  /* shareable memory left (SHARED claims) */
    uint32_t node;          /* owning node index */
    uint16_t share_cnt;     /* SHARED claims currently on this GPU */
    uint16_t rsvd;
} dra_gpu_rec;

#define DRA_GPU_MIG_ENABLED    0x01u  /* nvlib.go:152 / :316-318 — full GPU xor MIG parent */
#define DRA_GPU_FULL_ALLOCATED 0x02u
#define DRA_GPU_UNAVAILABLE    0x04u

/* One request.  Flat form of the legacy GpuClaimParameters / MigDeviceClaimParameters
 * (shapes survive only in demo/specs/mig+mps/sharing-demo-parameters.yaml:22-41 and
 * demo/specs/selectors/parameters.yaml:7-27) and of today's DeviceRequest + DeviceClass + CEL
 * `profile == '...'` + matchAttribute parentUUID (demo/specs/quickstart/gpu-test4.yaml:19-44). */
typedef struct dra_claim_rec {
    uint8_t  kind;          /* DRA_KIND_* */
    uint8_t  profile;       /* NVML GI profile enum (kind MIG) */
    uint16_t count;         /* devices wanted (kind GPU), else ignored */
    uint32_t node;          /* selectedNode (Allocate) — overridden per candidate in UnsuitableNodes */
    uint32_t mem_limit_mib; /* kind SHARED: MPS pinned-memory limit, sharing.go:234-237 arithmetic */
    uint32_t group;         /* != 0: consecutive MIG claims with equal group share one parent GPU */
} dra_claim_rec;

#define DRA_KIND_GPU    0u
#define DRA_KIND_MIG    1u
#define DRA_KIND_SHARED 2u

/* One allocated device (or one failed slot).  Bijective with the reference's device names
 * gpu-<index> / gpu-<parent>-mig-<profileId>-<start>-<size> (deviceinfo.go:74-80) that
 * DeviceRequestAllocationResult.Device carries (k8s types.go:795-840). */
typedef struct dra_out_rec {
    uint32_t gpu;           /* global inventory index, DRA_GPU_NONE when not allocated */
    uint8_t  start;
    uint8_t  size;
    uint8_t  profile;       /* MIG: claim profile; 0xFF GPU; 0xFE SHARED */
    uint8_t  status;        /* DRA_ST_* */
} dra_out_rec;

#define DRA_PROFILE_GPU    0xFFu
#define DRA_PROFILE_SHARED 0xFEu

#define DRA_ST_OK          0u
#define DRA_ST_NO_CAPACITY 1u
#define DRA_ST_BAD_PROFILE 2u
#define DRA_ST_GROUP       3u
#define DRA_ST_MEM_LIMIT   4u
#define DRA_ST_INVALID     5u
#define DRA_ST_POD         6u     /* pod mode (spec §12): the pod does not fit on the node; nothing of it was taken */
#define DRA_ST_SEARCH_LIMIT 7u    /* pod mode: the exhaustive search ran out of budget (DRA_EXH_BUDGET descents) */

/* One (model, profile) cell of the placement table: what getGpuInfo() collects from
 * GetGpuInstanceProfileInfo + GetGpuInstancePossiblePlacements (nvlib.go:244-295). */
typedef struct dra_prof_ent {
    uint8_t  size;          /* memory slices */
    uint8_t  rsvd;
    uint16_t start_mask;    /* bit s: placement {start s, size} is possible; 0 = profile not offered */
} dra_prof_ent;

typedef struct dra_profile_tbl {
    dra_prof_ent ent[DRA_MAX_PROFILES];
} dra_profile_tbl;

/* Per-GPU attributes a selector can test — the attributes GpuInfo.GetDevice publishes
 * (cmd/nvidia-dra-plugin/deviceinfo.go:102-132), interned to integers by the host.  spec §10. */
typedef struct dra_gpu_attr {
    uint32_t mem_total_mib;
    uint32_t cc;            /* cudaComputeCapability: major << 8 | minor */
    uint32_t index;
    uint16_t product;       /* host-interned productName id */
    uint16_t driver_major;
} dra_gpu_attr;

/* One instruction of a selector program (postfix, boolean stack).  Flat form of the legacy
 * GpuClaimParameters.spec.selector trees (demo/specs/selectors/parameters.yaml:7-27) and of the CEL subset
 * in demo/specs/quickstart/gpu-test6.yaml:23-31. */
typedef struct dra_sel_ins {
    uint8_t  op;            /* DRA_SEL_* */
    uint8_t  attr;          /* DRA_ATTR_* */
    uint8_t  cmp;           /* DRA_CMP_* */
    uint8_t  rsvd;
    uint32_t value;
} dra_sel_ins;

#define DRA_SEL_MAX_INS 8u
typedef struct dra_selector { dra_sel_ins ins[DRA_SEL_MAX_INS]; } dra_selector;

#define DRA_SEL_END 0u
#define DRA_SEL_CMP 1u
#define DRA_SEL_AND 2u
#define DRA_SEL_OR  3u
#define DRA_SEL_NOT 4u
#define DRA_ATTR_MEMORY_MIB   0u
#define DRA_ATTR_CC           1u
#define DRA_ATTR_INDEX        2u
#define DRA_ATTR_PRODUCT      3u
#define DRA_ATTR_DRIVER_MAJOR 4u
#define DRA_CMP_EQ 0u
#define DRA_CMP_NE 1u
#define DRA_CMP_LT 2u
#define DRA_CMP_LE 3u
#define DRA_CMP_GT 4u
#define DRA_CMP_GE 5u
#define DRA_CMP_IN_MASK 6u

/* ---- context ------------------------------------------------------------------------------------- */

typedef struct dra_ctx dra_ctx;

typedef struct dra_cfg {
    uint32_t abi_version;   /* DRA_ABI_VERSION */
    int32_t  device;        /* CUDA device ordinal */
    void*    stream;        /* cudaStream_t to run on; NULL = the context creates its own */
    uint32_t max_claims;    /* capacity hint; buffers grow on demand */
    uint32_t flags;         /* DRA_CFG_* */
} dra_cfg;

#define DRA_CFG_USE_GRAPH  0x1u  /* dra_allocate_batch: replay H2D -> kernels -> D2H as ONE CUDA graph launch when a
                                    call repeats the previous call's buffers and sizes (captured on the 2nd such call) */
#define DRA_CFG_NO_FUSED   0x2u  /* never take the single-launch path (always bucket + pack); for tests */
#define DRA_CFG_NO_DIRECT  0x4u  /* dra_allocate_batch: never let the single-launch kernel read the claims from / write the
                                    results to the pinned host buffers itself (direct host I/O, one cooperative launch);
                                    always use copy-engine transfers around the kernels */

#define DRA_CFG_RESIDENT   0x8u  /* dra_allocate_batch: keep the single-launch kernel RESIDENT and hand it batches by doorbell (a command
                                    line + sequence number in mapped host memory, completion word back) — no kernel launch, no stream
                                    call per batch.  Applies to batches that fit the staged single-launch form on an inventory of at most
                                    (SMs - 1) nodes with page-locked buffers; everything else stops the resident kernel first and takes
                                    the usual path.  The kernel leaves by itself after DRA_SERVE_IDLE_MS (20) ms without a batch. */

/* error codes (negative) */
#define DRA_OK        0
#define DRA_E_INVAL  (-1)
#define DRA_E_CUDA   (-2)
#define DRA_E_NCCL   (-3)
#define DRA_E_NOMEM  (-4)
#define DRA_E_STATE  (-5)

/* batch flags */
#define DRA_F_NODE_SORTED 0x1u  /* claims already grouped by ascending node (stable): skip bucketing.
                                   Verified on the device; violation -> DRA_E_INVAL, nothing changed */
#define DRA_F_FRESH_INVENTORY 0x2u  /* evaluate against the inventory as dra_set_inventory last loaded it
                                   (ignoring earlier batches); the result becomes the live inventory */

#define DRA_F_EXHAUSTIVE 0x4u   /* pod mode (spec §12): backtracking search over every valid (GPU, placement) of the pod's MIG
                                   claims — a pod fails only if NO assignment exists.  dra_allocate_pods_batch and
                                   dra_unsuitable_batch; the enumeration it searches is the one deviceLib.getGpuInfo builds
                                   (cmd/nvidia-dra-plugin/nvlib.go:244-295) */

int  dra_abi_version(void);

/* Creates a context bound to one CUDA device + one stream.  Fails with DRA_E_CUDA when no usable
 * sm_90 device exists — there is no CPU fallback. */
int  dra_ctx_create(const dra_cfg* cfg, dra_ctx** out);
void dra_ctx_destroy(dra_ctx* ctx);
const char* dra_last_error(const dra_ctx* ctx);      /* ctx may be NULL: last create error */

/* Placement table for one GPU model — replaces the per-GPU migProfiles list built by
 * deviceLib.getGpuInfo (cmd/nvidia-dra-plugin/nvlib.go:244-295). */
int  dra_set_placement_table(dra_ctx* ctx, uint32_t model, const dra_profile_tbl* tbl);

/* Inventory of every node this context serves — replaces the AllocatableDevices map published per node
 * (cmd/nvidia-dra-plugin/nvlib.go:111-180, driver.go:71-83) / the per-node NodeAllocationState CRD of
 * the classic driver.  gpus sorted by (node, local index); node_off has n_node+1 entries. Copied. */
int  dra_set_inventory(dra_ctx* ctx, const dra_gpu_rec* gpus, uint32_t n_gpu,
                       const uint32_t* node_off, uint32_t n_node);
/* Optional, spec §10: attributes of the same n_gpu GPUs (same order) and the selector table.  A claim names
 * its selector by 1-based id: kinds GPU and MIG in mem_limit_mib, kind SHARED in group. */
int  dra_set_gpu_attrs(dra_ctx* ctx, const dra_gpu_attr* attrs, uint32_t n_gpu);
int  dra_set_selectors(dra_ctx* ctx, const dra_selector* sels, uint32_t n_sel);
/* Read the live inventory back (n_gpu records). */
int  dra_get_inventory(dra_ctx* ctx, dra_gpu_rec* gpus, uint32_t n_gpu);
/* Restore the live inventory to what dra_set_inventory last loaded (device-side copy). */
int  dra_reset_inventory(dra_ctx* ctx);

/* Allocate(): stands in for  controller.Driver.Allocate(ctx, claims []*ClaimAllocation, selectedNode)
 * (k8s.io/dynamic-resource-allocation/controller, not vendored: vendor/modules.txt:757-760) batched over
 * many pods — every claim carries its selectedNode.  Mutates the context's inventory.
 *   claims[n_claim]           host memory
 *   out_off[n_claim] or NULL  first OutRec slot of each claim (NULL: slot i, all counts must be 1)
 *   out[n_out]                host memory, filled in input order
 * Per-claim failure is NOT an error (out[].status != 0), like the per-claim Error strings of
 * cmd/nvidia-dra-plugin/driver.go:126-137. */
int  dra_allocate_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                        const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, uint32_t flags);

/* Same, all pointers are DEVICE memory on ctx's device; enqueued on ctx's stream, returns without
 * synchronising (errors detected on the device surface at the next dra_ctx_sync). */
int  dra_allocate_batch_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                               const uint32_t* d_out_off, dra_out_rec* d_out, uint32_t n_out,
                               uint32_t flags);
int  dra_ctx_sync(dra_ctx* ctx);

/* UnsuitableNodes(): stands in for  controller.Driver.UnsuitableNodes(ctx, pod, claims, potentialNodes)
 * batched over pods.  Pure: evaluates each pod's claims on a snapshot of each candidate node.
 *   pod_off[n_pod+1]   claim range of each pod
 *   cand_off[n_pod+1]  range of each pod's candidates in cand_nodes
 *   suitable_bits      ceil(cand_off[n_pod]/8) bytes; bit k = k-th (pod,candidate) pair is suitable
 * Dense form: cand_nodes == NULL and cand_off == NULL evaluates every pod against EVERY node of the inventory
 * (pair k = pod * n_node + node; suitable_bits has ceil(n_pod*n_node/8) bytes) without any candidate arrays. */
int  dra_unsuitable_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                          const uint32_t* pod_off, uint32_t n_pod,
                          const uint32_t* cand_nodes, const uint32_t* cand_off,
                          uint8_t* suitable_bits, uint32_t flags /* 0 or DRA_F_EXHAUSTIVE (spec §12) */);

/* Allocate() with pod boundaries (spec §12): what the classic driver's Allocate did after UnsuitableNodes had found
 * an assignment for ALL of a pod's claims on the selected node (SURVEY App. A) — each pod (claims
 * pod_off[p] .. pod_off[p+1], all naming the same node, at most DRA_MAX_POD) is placed atomically; with
 * DRA_F_EXHAUSTIVE its MIG claims are placed by the backtracking search over the placement enumeration of
 * nvlib.go:244-295 (multi-request shape: demo/specs/quickstart/gpu-test4.yaml:19-44).  A pod that does not fit
 * takes nothing: its slots carry DRA_ST_POD (or DRA_ST_SEARCH_LIMIT).  The pods are sorted by node with
 * dra_allocate_batch's counting sort: n_pod > 0 on an inventory of 102,400 nodes or more is DRA_E_INVAL, refused
 * before anything runs.  Slots are counted from each claim's own fields (a GPU claim naming no node of the inventory has
 * one); slots no claim owns read back as 0.  pod_off not monotone or not spanning [0, n_claim], a slot range outside
 * n_out, or unknown flags: DRA_E_INVAL, refused before anything runs, with no output written and no state changed.
 * Host buffers; flags: DRA_F_EXHAUSTIVE, DRA_F_FRESH_INVENTORY. */
int  dra_allocate_pods_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                             const uint32_t* pod_off, uint32_t n_pod,
                             const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, uint32_t flags);

/* Choose the node and Allocate() in one call (spec §13): the batched form of the classic controller's "pending"
 * allocations — when it evaluated a pod for UnsuitableNodes it folded in the tentative assignments of the pods before
 * it (SURVEY App. A), so that two pods needing the last free slot of a node were not both sent there.  Pods are taken
 * in input order; pod p tries its candidates cand_nodes[cand_off[p] .. cand_off[p+1]) in list order, each evaluated
 * as in dra_allocate_pods_batch (spec §12, with DRA_F_EXHAUSTIVE the backtracking search) on that node's CURRENT state,
 * with every claim's node taken to be the candidate; the first candidate where the pod fits takes it.
 *   cand_nodes == cand_off == NULL   dense form: every pod against every node of the inventory, ascending
 *   pod_node[n_pod]                  the node each pod was placed on, 0xFFFFFFFF when none
 * A claim's own node field is ignored and never written.  A candidate naming no node of the inventory is skipped.  A
 * pod placed nowhere takes nothing: its slots carry DRA_ST_POD, or DRA_ST_SEARCH_LIMIT when any of its evaluations ran
 * out of budget (DRA_ST_INVALID for claims invalid by §3/§10); a pod of more than DRA_MAX_POD claims is INVALID; an
 * empty pod is skipped.  Slots are counted as if each claim named a node of the inventory.  With one candidate per pod,
 * the node its claims name, the result is byte for byte dra_allocate_pods_batch's.  pod_off / cand_off not monotone or
 * not spanning, a slot outside n_out, unknown flags, or candidates (cand_off[n_pod] > 0) on an inventory of 102,400
 * nodes or more (the pairs are sorted by node as dra_allocate_pods_batch's pods are; the dense form has no such limit):
 * DRA_E_INVAL, nothing changed.  Host buffers; flags: DRA_F_EXHAUSTIVE, DRA_F_FRESH_INVENTORY. */
int  dra_place_pods_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                          const uint32_t* pod_off, uint32_t n_pod,
                          const uint32_t* cand_nodes, const uint32_t* cand_off,
                          const uint32_t* out_off, dra_out_rec* out, uint32_t n_out,
                          uint32_t* pod_node, uint32_t flags);

/* Preemption (spec §14): for pods that fit nowhere, which lower-priority running pods to evict on each candidate node,
 * and which node to evict them on — kube-scheduler's DefaultPreemption (SelectVictimsOnNode, pickOneNodeForPreemption)
 * without start times; PodDisruptionBudgets through dra_preempt_pdb_batch.  Pure: nothing is written to the inventory. */
#define DRA_PRE_FITS         0u   /* the pod fits on the node as it is: no victims */
#define DRA_PRE_EVICT        1u   /* the pod fits once the victims are gone */
#define DRA_PRE_NO           2u   /* it does not fit even with every lower-priority pod gone (or: no such node) */
#define DRA_PRE_SEARCH_LIMIT 3u   /* an evaluation ran out of DRA_EXH_BUDGET */
#define DRA_PRE_INVALID      4u   /* more than DRA_MAX_POD claims, or a claim invalid by §3/§10 */

/* The running pods: the allocations the live inventory holds, as dra_deallocate_batch takes them (claims, out_off or
 * NULL, out[n_out]), split into pods by pod_off[n_pod+1].  Pod index order is start order, earliest first. */
typedef struct dra_running_pods {
    const dra_claim_rec* claims; uint32_t n_claim;
    const uint32_t* pod_off;     uint32_t n_pod;     /* n_pod + 1 entries */
    const int32_t*  prio;                             /* n_pod */
    const uint32_t* out_off;                          /* NULL: slot i, as dra_deallocate_batch */
    const dra_out_rec* out;      uint32_t n_out;
} dra_running_pods;

/* Pending pods as in dra_place_pods_batch (claims, pod_off, candidates or the dense form; each claim's node field is
 * ignored), with priority prio[p].  Per pair (n_pair = cand_off[n_pod], dense n_pod * n_node), each may be NULL:
 *   pair_status[k]   DRA_PRE_*          pair_victims[k]  victims of an EVICT pair, else 0
 * Per pod:
 *   pod_node[p]      the node chosen (FITS or EVICT), else 0xFFFFFFFF      pod_status[p]  DRA_PRE_*
 *   n_victims[p]     the chosen pair's victim count (always the full count)
 *   victims[p * max_victims + k]  its first min(n_victims[p], max_victims) victims as running-pod indices, in eviction
 *                    order (priority descending, then index); the rest of the row 0xFFFFFFFF.
 * DRA_E_INVAL with nothing written: unknown flags, pod_off / cand_off / running->pod_off not monotone or not spanning,
 * dense n_pod * n_node >= 2^32, a running slot range outside running->n_out, a running pod whose OK slots name a GPU
 * index >= n_gpu or GPUs of two nodes, max_victims > 0 without victims, running pods on an inventory of 102,400 nodes
 * or more (they are sorted by node as dra_allocate_pods_batch's pods are).  n_pod == 0 returns DRA_OK once flags, pod_off,
 * cand_off and max_victims pass, without examining the running pods.  Host buffers; flags: 0 or DRA_F_EXHAUSTIVE. */
int  dra_preempt_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                       const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                       const uint32_t* cand_nodes, const uint32_t* cand_off,
                       const dra_running_pods* running,
                       uint8_t* pair_status, uint32_t* pair_victims,
                       uint32_t* pod_node, uint8_t* pod_status, uint32_t* n_victims,
                       uint32_t* victims, uint32_t max_victims, uint32_t flags);

/* Disruption budgets (spec §14, "Disruption budgets"): PodDisruptionBudgets lowered by the caller.  Running pod r counts
 * against budget run_pdb[r] (at most one; DRA_PDB_NONE for none, also for a pod listed in its budget's DisruptedPods),
 * whose status.disruptionsAllowed is allowed[b].  NULL, n_pdb == 0 or every run_pdb DRA_PDB_NONE: no budgets. */
#define DRA_PDB_NONE 0xFFFFFFFFu
#define DRA_PDB_MAX_RUNNING (1u << 29)   /* with n_pdb > 0, fewer running pods than this (a violation count takes 29 bits) */
typedef struct dra_disruption_budgets {
    const uint32_t* run_pdb;   /* [running->n_pod]: budget of each running pod, DRA_PDB_NONE for none */
    const int32_t*  allowed;   /* [n_pdb]: disruptionsAllowed of each budget */
    uint32_t        n_pdb;
} dra_disruption_budgets;

/* dra_preempt_batch with disruption budgets (NULL: none): on each pair, V's members whose eviction would take their
 * budget below zero (counted over V in order, from allowed afresh for every pair) are reprieved first, then the others;
 * the pod's EVICT pair is the one with the fewest violating victims first, then dra_preempt_batch's order.  Victim rows
 * stay in V order.  Two more outputs, each may be NULL:
 *   pair_violations[k]  the violating victims of an EVICT pair, else 0
 *   pod_violations[p]   the chosen pair's (EVICT), else 0
 * With no budgets every output is byte for byte dra_preempt_batch's, every violation count 0.  DRA_E_INVAL with nothing
 * written: dra_preempt_batch's errors, n_pdb > 0 without allowed, and, when n_pod > 0: a run_pdb[r] neither DRA_PDB_NONE
 * nor below n_pdb, running pods with n_pdb > 0 and no run_pdb, n_pdb > 0 with DRA_PDB_MAX_RUNNING running pods or more.
 * n_pod == 0 returns DRA_OK without examining the running pods or run_pdb.  Host buffers. */
int  dra_preempt_pdb_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                           const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                           const uint32_t* cand_nodes, const uint32_t* cand_off,
                           const dra_running_pods* running, const dra_disruption_budgets* budgets,
                           uint8_t* pair_status, uint32_t* pair_victims, uint32_t* pair_violations,
                           uint32_t* pod_node, uint8_t* pod_status, uint32_t* n_victims, uint32_t* pod_violations,
                           uint32_t* victims, uint32_t max_victims, uint32_t flags);

/* Preempt and place (spec §15): dra_preempt_batch's question for a batch that sees itself, answered and applied.  Pods
 * are taken in input order; pod p is judged as dra_preempt_batch judges it, but on the inventory as the pods before it
 * left it (their placements held, their victims gone), with only the running pods no earlier pod evicted as possible
 * victims; the pods of the call are never victims.  Its choice is then applied: for EVICT the victims are released from
 * the live inventory as dra_deallocate_batch releases them; for FITS or EVICT the pod is allocated on the chosen node as
 * dra_allocate_pods_batch allocates it, OutRecs written.  The result is byte for byte the host loop, per pod:
 * dra_preempt_batch with that one pod and the running pods not yet evicted, dra_deallocate_batch of its victims,
 * dra_allocate_pods_batch of its claims on the chosen node.
 *   claims / pod_off / prio / candidates   as dra_preempt_batch (cand_nodes == cand_off == NULL: dense form); each
 *                    claim's node field is ignored and never written
 *   running          the running pods, as dra_preempt_batch takes them
 *   out_off / out[n_out]  as dra_place_pods_batch: slots counted as if each claim named a node of the inventory
 *   pod_node[p]      the node chosen (FITS or EVICT), else 0xFFFFFFFF     pod_status[p]  DRA_PRE_*
 *   evicted_by[r]    the pod that evicted running pod r, else 0xFFFFFFFF (each pod's victims in eviction order:
 *                    priority descending, then index)
 * A pod placed nowhere takes nothing: its slots carry DRA_ST_SEARCH_LIMIT when its status is DRA_PRE_SEARCH_LIMIT, else
 * DRA_ST_POD (DRA_ST_INVALID for claims invalid by §3/§10, every claim of a pod of more than DRA_MAX_POD).  A pod with
 * a claim invalid in the call's slot mode (without out_off, a GPU claim of count != 1) is DRA_PRE_INVALID and evicts
 * nothing.  An empty pod is FITS on its first candidate naming a node, with nothing written.  The call RELEASES THE
 * VICTIMS ITSELF: their allocations are gone from the live inventory when it returns, so the caller must not pass them
 * to dra_deallocate_batch again.  DRA_E_INVAL, with no output and no inventory word written: unknown flags, pod_off /
 * cand_off / running->pod_off not monotone or not spanning, more than 2^30 - 1 candidates for a pod or nodes in the
 * inventory, dense n_pod * n_node >= 2^32, a pending slot outside n_out, a running slot range outside running->n_out, a
 * running pod whose OK slots name a GPU index >= n_gpu or GPUs of two nodes, running pods or candidates (cand_off[n_pod]
 * > 0) on an inventory of 102,400 nodes or more (both are sorted by node).  n_pod == 0 returns DRA_OK after the
 * checks of the pending arrays, without examining the running pods.  Host buffers; flags: 0 or DRA_F_EXHAUSTIVE. */
int  dra_preempt_place_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                             const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                             const uint32_t* cand_nodes, const uint32_t* cand_off,
                             const dra_running_pods* running,
                             const uint32_t* out_off, dra_out_rec* out, uint32_t n_out,
                             uint32_t* pod_node, uint8_t* pod_status, uint32_t* evicted_by, uint32_t flags);

/* Pod capacity (spec §16): how many copies of each pod every candidate node still takes — the question asked about a
 * workload rather than a pod (replicas of a Deployment that fit and where, an autoscaler's simulation, "free 3g.40gb
 * instances per node", a figure to order dra_place_pods_batch's candidates by).  Pure: nothing is written to the
 * inventory.  Pods and candidates as dra_unsuitable_batch takes them (cand_nodes == cand_off == NULL: dense form, pair
 * k = pod * n_node + node); each claim's node field is ignored.  For pair k = (pod, node): the pod is evaluated on a
 * private copy of the node as dra_allocate_pods_batch evaluates it with the same flags (spec §12, slots as if out_off
 * were given: a GPU claim may have count up to DRA_MAX_COUNT), the placement kept each time it succeeds, until an
 * evaluation fails or max_copies (1 .. 65535) copies are placed.
 *   pair_copies[k]   copies placed: the number of OK pods dra_allocate_pods_batch gives for max_copies identical copies
 *                    of the pod naming that node.  With DRA_F_EXHAUSTIVE, >= 1 exactly when dra_unsuitable_batch sets
 *                    the pair's bit with that flag; without it the evaluation is §12's, not §8's claim walk.
 *   pair_stop[k]     (may be NULL) why counting stopped: DRA_ST_OK max_copies reached (the count is "at least");
 *                    DRA_ST_POD the next copy does not fit; DRA_ST_SEARCH_LIMIT the next copy's search ran out of
 *                    DRA_EXH_BUDGET (the count is a lower bound); DRA_ST_INVALID more than DRA_MAX_POD claims or a claim
 *                    invalid by §3/§10 (copies 0)
 *   pod_total[p]     (may be NULL) the sum of the pod's pair_copies: with each node listed once, the copies the whole
 *                    candidate set takes (nodes are independent); a node listed twice is counted twice
 *   pod_nodes[p]     (may be NULL) how many of the pod's pairs take at least one copy
 * A candidate naming no node of the inventory: copies 0, DRA_ST_POD.  Otherwise an empty pod: copies max_copies,
 * DRA_ST_OK.  DRA_E_INVAL with nothing written: unknown flags, max_copies 0 or above 65535, pod_off / cand_off not
 * monotone or not spanning, dense n_pod * n_node >= 2^32, pair_copies NULL with pairs to answer.  n_pod == 0 returns
 * DRA_OK after those checks.  On a sharded world the call is exact on any rank after dra_shard_sync_inventory_device,
 * which makes that rank's live copy the world's state; dra_pod_capacity_batch_global_device answers across the ranks
 * without the sync, each rank counting the pairs of its own nodes.  Host buffers; flags: 0 or DRA_F_EXHAUSTIVE. */
int  dra_pod_capacity_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                            const uint32_t* pod_off, uint32_t n_pod,
                            const uint32_t* cand_nodes, const uint32_t* cand_off,
                            uint32_t max_copies,
                            uint16_t* pair_copies, uint8_t* pair_stop,
                            uint64_t* pod_total, uint32_t* pod_nodes, uint32_t flags);

/* Deallocate(): stands in for controller.Driver.Deallocate(ctx, claim).  Inverse update from the
 * claims and the OutRecs dra_allocate_batch produced for them (same out_off convention), or any other records: a MIG
 * record frees ((1 << size) - 1) << start cut to 16 bits, nothing when start >= 16 (spec §9).  Every claim's slot range
 * is checked before anything is enqueued: one that leaves [0, n_out), or n_out < n_claim without out_off, returns
 * DRA_E_INVAL with nothing launched and the inventory unchanged. */
int  dra_deallocate_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim,
                          const uint32_t* out_off, const dra_out_rec* out, uint32_t n_out);

/* ---- multi-GPU (one process per GPU; nodes are sharded whole) ------------------------------------ */

/* 128-byte NCCL unique id, generated on rank 0 and handed to the other ranks by the host runtime. */
int  dra_comm_unique_id(void* id128);
int  dra_comm_init(dra_ctx* ctx, const void* id128, int rank, int world);
/* dra_allocate_batch_device on this rank's claims, then ONE ncclAllGather of n_per_rank OutRecs per rank
 * into d_out_all[world * n_per_rank] on the same stream (slots past this rank's n_out are zero-filled). */
int  dra_allocate_batch_gather_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                      const uint32_t* d_out_off, dra_out_rec* d_out_all,
                                      uint32_t n_out, uint32_t n_per_rank, uint32_t flags);

/* The complete table of the last gather: device pointer (valid until the second-next gather call) and the
 * padded per-rank length; with the peer all-gather set up d_out_all may be NULL and this is the result. */
int  dra_gather_table(dra_ctx* ctx, const dra_out_rec** d_table, uint32_t* n_per_rank);
/* Device -> host read of the first n_rec records of that table on ctx's stream, then synchronises. */
int  dra_gather_read(dra_ctx* ctx, dra_out_rec* out_all, uint32_t n_rec);

/* Peer-memory all-gather (OutRecs as self-validating 16-byte packets over NVLink, no fence / flag; measurements in
 * profiles/peer_bench_r02.txt) — when set up, dra_allocate_batch_gather_device uses it instead of ncclAllGather.  Call after dra_comm_init on every rank:
 *   dra_peer_export(ctx, n_per_rank, handle)   allocates this rank's gather buffer, returns its 64-byte
 *                                              cudaIpcMemHandle_t;  the host runtime all-gathers the handles;
 *   dra_peer_import(ctx, handles)              world * 64 bytes, in rank order.
 * Requires all ranks on one node with P2P access; on failure the NCCL path stays in use.  Every rank must export alike (the
 * same sizes, dra_set_shard_pairs, dra_set_shard_place, dra_set_shard_preempt, dra_set_shard_capacity, dra_set_shard_preempt_place and, for dra_shard_export, inventory size): each rank addresses its peers' buffers by its
 * own layout, so dra_peer_import / dra_peer_import_local refuse a peer set up differently with DRA_E_INVAL.
 * dra_peer_export(ctx, 0, NULL) switches the peer path off again. */
int  dra_peer_export(dra_ctx* ctx, uint32_t n_per_rank, void* handle64);
int  dra_peer_import(dra_ctx* ctx, const void* handles);

/* The same mapping for contexts of ONE process (one Go driver process driving all GPUs of a box, or tests): instead of
 * NCCL + IPC handles, call dra_comm_init_local(ctx, rank, world) on every context, dra_peer_export / dra_shard_export
 * (handle may be NULL), then dra_peer_import_local(ctx, ctxs) with the world contexts in rank order (peer access between
 * their devices is enabled here).  Calls of different ranks must then be issued without waiting for each other.
 * One context per DEVICE is the supported layout; several ranks on one device work for batches that take the
 * single-launch kernel (the tests do it) but can starve each other on the sort path (a waiting gather holds the SMs). */
int  dra_comm_init_local(dra_ctx* ctx, int rank, int world);
int  dra_peer_import_local(dra_ctx* ctx, dra_ctx* const* ctxs);

/* Cross-rank rendezvous ON THE DEVICE: enqueues one tiny kernel on the context's stream that tells every peer "rank r is
 * here" (one 4-byte store over NVLink each) and waits until every peer has said the same (after dra_peer_import /
 * dra_peer_import_local; every rank must call it the same number of times; no host synchronisation, returns at once).
 * It orders nothing but time: the ranks' streams leave it within one NVLink latency of each other.  bench.py calls it
 * between its untimed L2 flush and the timed step, so that a rank's step does not absorb its peers' flush-time skew.
 * A peer that never arrives within DRA_PEER_TIMEOUT_MS sets the context's error flag (next call: DRA_E_STATE). */
int  dra_peer_rendezvous_device(dra_ctx* ctx);

/* ---- sharded GLOBAL batch (BASELINE configs[2]: one batch, claim x node space sharded over the GPUs of a box) -----
 * Every rank loads the WHOLE inventory (dra_set_inventory) and serves a contiguous node range
 * (dra_set_shard; pool = node, nodes are never split: vendor/k8s.io/dynamic-resource-allocation/kubeletplugin/
 * draplugin.go:427-435).  dra_allocate_batch_global_device takes the SAME global claim array on every rank: the rank
 * filters the claims of its nodes on the device (stable compaction in input order), allocates them, and writes each
 * OutRec at the claim's GLOBAL slot of every rank's result table — the path's one collective, an all-gather done as
 * 16-byte self-validating packets over NVLink inside the allocation kernel (no host partition / merge, no un-permute).
 * Claims that name no node are answered by the rank with take_stray != 0 (exactly one rank).
 *   dra_shard_export(ctx, n_out_max, cap_per_rank, handle)  allocates table + staging (cap_per_rank = upper bound of the
 *        OutRec slots one rank can own, 0 = n_out_max); handles are exchanged and mapped with dra_peer_import as above
 *   result: dra_gather_table / dra_gather_read (n_out records, input order, global GPU indices)
 * out_off must tile [0, n_out) (slots no claim owns keep their previous contents).  flags: DRA_F_FRESH_INVENTORY.
 * With world == 1 no export is needed (the table is local).  A rank's live inventory is authoritative for its own
 * node range only (UnsuitableNodes and pods Allocate on such a world: dra_unsuitable_batch_global_device and
 * dra_allocate_pods_batch_global_device below; the whole world's state on every rank: dra_shard_sync_inventory_device;
 * Deallocate: dra_deallocate_batch_global_device).  d_claims may also be a pinned host buffer (dra_host_alloc): the compaction kernel reads every claim
 * exactly once, so it then ingests the batch over PCIe itself — no copy-engine transfer in front of the call. */
int  dra_set_shard(dra_ctx* ctx, uint32_t node_lo, uint32_t node_hi, int take_stray);
/* The whole partition: rank r serves nodes [bounds[r], bounds[r+1]) (bounds has world+1 entries, bounds[world] = n_node),
 * stray_rank answers claims naming no node.  Since every rank reads the whole claim array, it then also COUNTS what every
 * rank will answer — receivers know how many records to expect from each peer before the first one arrives, and the gather
 * runs without any header or completion round.  Preferred over dra_set_shard whenever world > 1. */
int  dra_set_shard_map(dra_ctx* ctx, const uint32_t* bounds, int stray_rank);
int  dra_shard_export(dra_ctx* ctx, uint32_t n_out_max, uint32_t cap_per_rank, void* handle64);
int  dra_allocate_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                      const uint32_t* d_out_off, uint32_t n_out, uint32_t flags);

/* Sharded UnsuitableNodes.  After sharded Allocate calls a rank's inventory is stale outside its node range, so
 * dra_unsuitable_batch on one rank cannot answer for the whole world; this call can.  Each rank evaluates only the pairs
 * whose candidate node lies in its range, on its live inventory, and the ranks exchange their bits over peer memory.
 *
 * Room for the bit exchange in the buffer dra_shard_export maps.  World > 1: call before dra_shard_export (afterwards:
 * DRA_E_STATE); every rank with the same max_pairs.  The export then also sizes the call's scratch for max_pairs (about
 * 4 bytes per pair beyond the staging), so that no call reallocates while its peers wait.  World 1 needs no call (buffers
 * grow on demand). */
int  dra_set_shard_pairs(dra_ctx* ctx, uint32_t max_pairs);
/* UnsuitableNodes over a sharded world (spec §8 / §12).  The SAME pods and candidates on every rank (device pointers, or
 * dra_host_alloc'ed buffers).  A pair is decided by the rank whose node range holds its candidate node, against that rank's
 * live inventory; a candidate that names no node of the inventory is unsuitable.  Every rank ends with the WHOLE bitmap in
 * d_suitable_bits: exactly ceil(n_pair/8) bytes, bits past n_pair zero.  Dense form = cand_nodes == cand_off == NULL
 * (pair = pod * n_node + node, n_pair = n_pod * n_node).  Enqueues on ctx's stream and returns; completion and
 * device-detected errors (pod_off / cand_off not monotone or not spanning their arrays: DRA_E_INVAL, every bit zero) surface
 * at dra_ctx_sync.  Every rank must make the same calls.  flags: 0 or DRA_F_EXHAUSTIVE. */
int  dra_unsuitable_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                        const uint32_t* d_pod_off, uint32_t n_pod,
                                        const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                        uint8_t* d_suitable_bits, uint32_t flags);

/* Pods Allocate over a sharded world (spec §12, "Sharded form"): the classic flow's second step after
 * dra_unsuitable_batch_global_device(..., DRA_F_EXHAUSTIVE).  The SAME claims, pod_off, out_off, n_out and flags on every
 * rank (device pointers, or dra_host_alloc'ed buffers).  A non-empty pod belongs to the rank whose node range holds the
 * node of its FIRST claim (a node outside the inventory: the stray rank); the owner writes every slot of every claim of the
 * pod (OK, POD, SEARCH_LIMIT or INVALID, validated and counted on global node indices) and applies the placements to its
 * live inventory.  Every rank ends with the WHOLE table (dra_gather_table / dra_gather_read: n_out records, global slots,
 * global GPU indices): byte for byte what dra_allocate_pods_batch answers on ONE inventory made of every rank's own nodes,
 * and each rank's inventory over its own GPU range equals that call's; GPUs outside the range are not written.
 * flags: DRA_F_EXHAUSTIVE, DRA_F_FRESH_INVENTORY (the pristine copy of the rank's own GPUs is read, the live one written).
 * Prerequisites as for dra_allocate_batch_global_device, except that world > 1 needs dra_set_shard_map (a bare
 * dra_set_shard: DRA_E_STATE).  Enqueues on ctx's stream and returns; n_pod == 0 enqueues nothing.  Completion and device-detected errors
 * surface at dra_ctx_sync: pod_off not monotone or not spanning [0, n_claim], a slot range outside n_out, or a rank owning
 * more slots than its packet room give DRA_E_INVAL on EVERY rank (they read the same arrays), with no inventory changed. */
int  dra_allocate_pods_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                           const uint32_t* d_pod_off, uint32_t n_pod,
                                           const uint32_t* d_out_off, uint32_t n_out, uint32_t flags);

/* Room for the sharded place-pods call's replicated pod states (8 bytes per pod, plus 64) in the buffer dra_shard_export
 * maps.  World > 1: call before dra_shard_export (afterwards: DRA_E_STATE), every rank with the same max_pods; the peer
 * import refuses a peer set up differently.  Load the inventory first: the export then also sizes the call's sort for it,
 * so that no call frees a buffer (which waits for the whole device) while a peer's walk waits for it.  World 1 needs no
 * call. */
int  dra_set_shard_place(dra_ctx* ctx, uint32_t max_pods);
/* Place pods over a sharded world (spec §13, "Sharded form"): dra_place_pods_batch applied to the world's state.  The SAME
 * claims, pod_off, candidates (cand_nodes == cand_off == NULL and n_pair == 0: the dense form), out_off, n_out and flags on
 * every rank (device pointers, or dra_host_alloc'ed buffers).  Each rank evaluates the visits to its own nodes, on its live
 * inventory, and the ranks hand pods to each other through replicated state words.  Every rank ends with the WHOLE table
 * (dra_gather_table / dra_gather_read) and the whole d_pod_node[n_pod]: byte for byte what dra_place_pods_batch answers on
 * ONE inventory made of every rank's own nodes; each rank's own GPU range ends as that call leaves it, and no rank writes
 * a GPU record outside its range, live or pristine.  flags: DRA_F_EXHAUSTIVE, DRA_F_FRESH_INVENTORY (each rank starts its
 * own range from the pristine copy).  Prerequisites as for dra_allocate_pods_batch_global_device, plus n_pod <= the
 * max_pods of dra_set_shard_place at world > 1 (else DRA_E_STATE); world 1 (dra_set_shard(ctx, 0, n_node, 1)) needs no
 * export and answers exactly as dra_place_pods_batch.  Enqueues on ctx's stream and returns; n_pod == 0 enqueues nothing.
 * Completion and device-detected errors surface at dra_ctx_sync: pod_off / cand_off not monotone or not spanning their
 * arrays, more than 2^30 - 1 candidates for a pod, a slot range outside n_out, or a rank that could finalise more slots
 * than its packet room give DRA_E_INVAL on EVERY rank with no inventory changed; a peer that stops making progress gives
 * DRA_E_NCCL once nothing moved anywhere in the world for DRA_PEER_TIMEOUT_MS. */
int  dra_place_pods_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                        const uint32_t* d_pod_off, uint32_t n_pod,
                                        const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                        const uint32_t* d_out_off, uint32_t n_out, uint32_t* d_pod_node, uint32_t flags);

/* Room for the sharded preemption call in the buffer dra_shard_export maps: each rank's per-pod partials (32 bytes plus a
 * row of max_victims words, padded to 16 bytes) and its pairs' results (8 bytes a pair), one slice per rank and call parity.
 * World > 1: call before dra_shard_export (afterwards: DRA_E_STATE), every rank with the same sizes; the peer import refuses
 * a peer set up differently.  Load the inventory first: the export then also sizes the call's sort for it and its scratch
 * for max_pairs, so that no call frees a buffer (which waits for the whole device) while a peer waits for it.  World 1
 * needs no call. */
int  dra_set_shard_preempt(dra_ctx* ctx, uint32_t max_pods, uint32_t max_pairs, uint32_t max_victims);
/* Preemption over a sharded world (spec §14, "Sharded form"): dra_preempt_batch answered on the world's state.  The SAME
 * pending pods (claims, pod_off, prio), candidates (cand_nodes == cand_off == NULL: the dense form, n_pair = n_pod * n_node),
 * running pods, max_victims and flags on every rank (device pointers, or dra_host_alloc'ed buffers; `running` itself is a
 * host struct whose pointers are device-visible).  A pair is judged by the rank whose node range holds its candidate node,
 * against that rank's live inventory; a candidate naming no node of the inventory is DRA_PRE_NO.  Every rank ends with the
 * WHOLE outputs, laid out as dra_preempt_batch's, byte for byte what that call answers on ONE inventory made of every
 * rank's own nodes; d_pair_status / d_pair_victims may be NULL.  Nothing is written to any inventory, live or pristine.
 * world > 1 needs dra_set_shard_map (a bare dra_set_shard: DRA_E_STATE), dra_shard_export after dra_set_shard_preempt, and
 * dra_peer_import / dra_peer_import_local (else DRA_E_STATE); n_pod, n_pair and max_victims above its sizes: DRA_E_INVAL.
 * World 1 needs none of it and judges every node.  Host-side argument errors return before anything is enqueued.  Enqueues
 * on ctx's stream and returns; n_pod == 0 enqueues nothing.  Completion and device-detected errors surface at
 * dra_ctx_sync: pod_off / cand_off not monotone or not spanning their arrays, or the running pods' faults of
 * dra_preempt_batch give DRA_E_INVAL on EVERY rank with none of the outputs written; a peer that does not arrive within
 * DRA_PEER_TIMEOUT_MS gives DRA_E_NCCL.  flags: 0 or DRA_F_EXHAUSTIVE. */
int  dra_preempt_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                     const uint32_t* d_pod_off, const int32_t* d_prio, uint32_t n_pod,
                                     const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                     const dra_running_pods* running,
                                     uint8_t* d_pair_status, uint32_t* d_pair_victims,
                                     uint32_t* d_pod_node, uint8_t* d_pod_status, uint32_t* d_n_victims,
                                     uint32_t* d_victims, uint32_t max_victims, uint32_t flags);
/* dra_preempt_batch_global_device with disruption budgets, as dra_preempt_pdb_batch answers them: `budgets` (NULL: none)
 * is a host struct whose pointers are device-visible, the SAME on every rank; d_pair_violations and d_pod_violations may
 * be NULL.  The sizes of dra_set_shard_preempt are unchanged: the violation counts share the partials' and the pair
 * results' words.  Host-side, before anything is enqueued: n_pdb > 0 without allowed, and with n_pod > 0 running pods
 * with n_pdb > 0 and no run_pdb, or DRA_PDB_MAX_RUNNING running pods or more, give DRA_E_INVAL.  A run_pdb[r] neither
 * DRA_PDB_NONE nor below n_pdb is a running-pod fault: DRA_E_INVAL on EVERY rank at dra_ctx_sync, no output written.
 * With no budgets every output is byte for byte dra_preempt_batch_global_device's. */
int  dra_preempt_pdb_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                         const uint32_t* d_pod_off, const int32_t* d_prio, uint32_t n_pod,
                                         const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                         const dra_running_pods* running, const dra_disruption_budgets* budgets,
                                         uint8_t* d_pair_status, uint32_t* d_pair_victims, uint32_t* d_pair_violations,
                                         uint32_t* d_pod_node, uint8_t* d_pod_status, uint32_t* d_n_victims,
                                         uint32_t* d_pod_violations, uint32_t* d_victims, uint32_t max_victims, uint32_t flags);

/* Room for the sharded pod-capacity call in the buffer dra_shard_export maps: each rank's slice holds a 16-byte header,
 * then a u16 count and a u8 stop per pair, each part padded to 16 bytes, so 16 * (1 + ceil(max_pairs / 8) +
 * ceil(max_pairs / 16)) bytes, one slice per rank and call parity: world * 2 slices per rank (about 61 MB for 1.28 M pairs
 * at world 8).  World > 1: call before dra_shard_export (afterwards: DRA_E_STATE), every rank with the same max_pairs; the
 * peer import refuses a peer set up differently.  The export also sizes the call's scratch for max_pairs (one slice and 4
 * bytes a pair), so that no call frees a buffer while a peer waits for it.  World 1 needs no call. */
int  dra_set_shard_capacity(dra_ctx* ctx, uint32_t max_pairs);
/* Pod capacity over a sharded world (spec §16, "Sharded form"): dra_pod_capacity_batch answered on the world's state.  The
 * SAME claims, pod_off, candidates (cand_nodes == cand_off == NULL: the dense form, n_pair = n_pod * n_node), max_copies and
 * flags on every rank (device pointers, or dra_host_alloc'ed buffers).  A pair is counted by the rank whose node range
 * holds its candidate node, against that rank's live inventory; a candidate naming no node of the inventory gets 0 copies
 * and DRA_ST_POD.  Every rank ends with the WHOLE outputs, laid out as dra_pod_capacity_batch's, byte for byte what that
 * call answers on ONE inventory made of every rank's own nodes; d_pair_stop, d_pod_total and d_pod_nodes may be NULL.
 * Nothing is written to any inventory, live or pristine.  Needs dra_set_shard (else DRA_E_STATE); world > 1 needs
 * dra_set_shard_map spanning the inventory (a bare dra_set_shard: DRA_E_STATE), dra_shard_export after
 * dra_set_shard_capacity with max_pairs > 0 (even for a call with no pairs), and dra_peer_import /
 * dra_peer_import_local (else DRA_E_STATE).  World 1 needs no export,
 * counts every node, and answers byte for byte as dra_pod_capacity_batch.  Host-side argument errors (DRA_E_INVAL) return
 * before anything is enqueued: unknown flags, max_copies outside [1, 65535], one candidate array without the other, a
 * dense n_pair other than n_pod * n_node, n_pair above 2^32 - 16 or (world > 1) above max_pairs, n_pod above 2^26, NULL
 * d_pair_copies with pairs to answer.  Enqueues on ctx's stream and returns; n_pod == 0 enqueues nothing.  Completion and
 * device-detected errors surface at dra_ctx_sync: pod_off / cand_off not monotone or not spanning their arrays give
 * DRA_E_INVAL on EVERY rank with none of the outputs written; a peer that does not arrive within DRA_PEER_TIMEOUT_MS
 * gives DRA_E_NCCL, also with nothing written.  flags: 0 or DRA_F_EXHAUSTIVE. */
int  dra_pod_capacity_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                          const uint32_t* d_pod_off, uint32_t n_pod,
                                          const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                          uint32_t max_copies,
                                          uint16_t* d_pair_copies, uint8_t* d_pair_stop,
                                          uint64_t* d_pod_total, uint32_t* d_pod_nodes, uint32_t flags);

/* Every rank's live inventory becomes the world's state: for each GPU, the record its owning rank holds (the rank whose
 * node range contains the GPU's node, per the current dra_set_shard_map).  Own range untouched, pristine copy untouched.
 * Afterwards dra_get_inventory on any rank returns the whole world, and dra_set_shard_map may move node ranges between
 * ranks without losing allocations.  Every rank must make the call; enqueues on ctx's stream and returns; completion and
 * device-detected errors surface at dra_ctx_sync (a peer that never arrives within DRA_PEER_TIMEOUT_MS: DRA_E_NCCL, and
 * no record was copied).  world == 1: DRA_OK, nothing enqueued.
 * Prerequisites, each DRA_E_STATE with nothing enqueued: world > 1 needs dra_set_shard_map (a bare dra_set_shard is
 * refused); dra_shard_export, then dra_peer_import or dra_peer_import_local; the inventory loaded BEFORE the export (which
 * reserves n_gpu x 16 bytes of staging per call parity) and not grown since.
 * One process driving several ranks: dra_set_shard_map and dra_get_inventory synchronise the context's stream, so enqueue
 * the sync on EVERY rank before calling either on any rank; otherwise that rank's stream waits for peers whose call the
 * blocked thread has not made yet, and the sync times out. */
int dra_shard_sync_inventory_device(dra_ctx* ctx);

/* Room for the sharded preempt-and-place call: at most max_pods pending pods, max_pairs judged pairs (n_pair in the
 * candidate form, n_pod * n_node in the dense form) and max_run running pods per call.  World > 1: call before
 * dra_shard_export (afterwards: DRA_E_STATE), every rank with the same sizes; the peer import refuses a peer set up
 * differently.  Load the inventory first: the export then loads every kernel of the call and sizes its scratch (about
 * 16 bytes per GPU, 40 bytes per pair, 40 per pod and running pod) and its sort, so that no call loads a module or frees a
 * buffer while a peer waits for it.  World 1 needs no call. */
int dra_set_shard_preempt_place(dra_ctx* ctx, uint32_t max_pods, uint32_t max_pairs, uint32_t max_run);
/* Preempt and place over a sharded world (spec §15, "Sharded form"): dra_preempt_place_batch applied to the world's state,
 * the inventory made of every rank's own node range as that rank holds it.  The SAME claims, pod_off, prio, candidates
 * (cand_nodes == cand_off == NULL and n_pair == 0: the dense form), running pods, out_off, n_out and flags on every rank
 * (device pointers, or dra_host_alloc'ed buffers; `running` itself is a host struct whose pointers are device-visible).
 * Every rank ends with the WHOLE table (dra_gather_table / dra_gather_read: n_out records) and the whole d_pod_node[n_pod],
 * d_pod_status[n_pod] and d_evicted_by[running->n_pod]: byte for byte what dra_preempt_place_batch answers on that one
 * inventory.  Each rank's own GPU range ends as that call leaves it (the victims are released by the call); no rank writes
 * a GPU record outside its range, and none touches the pristine copy.  The ranks exchange their own ranges once, through
 * the inventory sync's staging, and then every rank runs the §15 walk on a private copy of the world's state.
 * Prerequisites as for dra_place_pods_batch_global_device: dra_set_shard (world 1: every node is the rank's) or, world > 1,
 * dra_set_shard_map; dra_set_shard_preempt_place and the inventory loaded before dra_shard_export; dra_peer_import or
 * dra_peer_import_local (else DRA_E_STATE).  n_pod, pairs or running pods above the reserved sizes, n_out above the exported
 * table: DRA_E_INVAL.  World 1 needs no export.  Host-side argument errors return before anything is enqueued.  Enqueues on
 * ctx's stream and returns; n_pod == 0 enqueues nothing.  Completion and device-detected errors surface at dra_ctx_sync:
 * pod_off / cand_off not monotone or not spanning their arrays, more than 2^30 - 1 candidates for a pod, a pending slot
 * outside n_out, or the running pods' faults of dra_preempt_place_batch give DRA_E_INVAL on EVERY rank, with no output
 * and no inventory word written; a peer that does not deliver its range within DRA_PEER_TIMEOUT_MS gives DRA_E_NCCL on
 * EVERY rank, also with nothing written (after the exchange the ranks agree on one verdict: the call fails everywhere or
 * nowhere).  The table is this context's own buffer, written by no peer; after a failed call its contents are undefined.
 * flags: 0 or DRA_F_EXHAUSTIVE. */
int dra_preempt_place_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                          const uint32_t* d_pod_off, const int32_t* d_prio, uint32_t n_pod,
                                          const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                          const dra_running_pods* running, const uint32_t* d_out_off, uint32_t n_out,
                                          uint32_t* d_pod_node, uint8_t* d_pod_status, uint32_t* d_evicted_by, uint32_t flags);

/* Deallocate over a sharded world (spec §9, "Sharded form"): the classic flow's last step.  The SAME claims, out_off and
 * OutRecs on every rank (device pointers, or dra_host_alloc'ed buffers; d_out may be the table dra_gather_table returns).
 * slots(c) is counted as by dra_deallocate_batch, on the whole inventory's node indices.  A rank applies only the OK slots
 * whose gpu lies in its own GPU range [node_off[node_lo], node_off[node_hi]) of dra_set_shard / dra_set_shard_map, and
 * writes no other GPU record (the pristine copy neither).  When every rank makes the call, every rank's own range ends as
 * dra_deallocate_batch would leave the world's state; dra_shard_sync_inventory_device then gives every rank that state.
 * Do NOT run dra_deallocate_batch on every rank with gathered records instead: it writes every GPU the records name, and a
 * SHARED slot on another rank's GPU wraps that copy's share count.
 * All or nothing: every claim's slot range [base, base + slots) is checked on the device before any record is applied; one
 * outside [0, n_out) gives DRA_E_INVAL at dra_ctx_sync on every rank, with no inventory word changed.
 * No exchange: no dra_shard_export or peer import is needed, the call waits for no peer, and it allocates nothing.  World 1
 * with dra_set_shard(0, n_node, 1) makes it a device-side, all-or-nothing dra_deallocate_batch of the whole inventory.
 * Prerequisites, each DRA_E_STATE with nothing enqueued: dra_set_inventory, and a shard (dra_set_shard or
 * dra_set_shard_map).  DRA_E_INVAL with nothing enqueued: NULL d_claims or d_out with n_claim > 0, n_out < n_claim
 * without out_off, n_claim or n_out above 2^26.  n_claim == 0: DRA_OK, nothing enqueued.  Otherwise two kernels are
 * enqueued on ctx's stream and the call returns; completion surfaces at dra_ctx_sync. */
int dra_deallocate_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                       const uint32_t* d_out_off, const dra_out_rec* d_out, uint32_t n_out);

/* ---- adjacent integer searches of the reference, batched (API completeness; SURVEY §8f-4) -------------- */

/* limit.Megabyte() over n quantities (api/nvidia.com/resource/gpu/v1alpha1/sharing.go:234-237):
 * mib[i] = bytes[i]/1024/1024 truncated toward zero, valid[i] = mib[i] > 0. */
int  dra_mps_limits_batch(dra_ctx* ctx, const int64_t* bytes, uint32_t n, int64_t* mib, uint8_t* valid);
/* imexDomainOffsets.add's search over n_dom domains (cmd/nvidia-dra-controller/imex.go:336-349): used offsets of
 * domain d are used[dom_off[d] .. dom_off[d+1]); out[d] = lowest multiple of step below limit not in them, -1 if none. */
int  dra_imex_offsets_batch(dra_ctx* ctx, const int32_t* used, const uint32_t* dom_off, uint32_t n_dom,
                            int32_t step, int32_t limit, int32_t* out);

/* One-time calibration (optional): measures, on this device and the loaded inventory, up to which batch size the
 * single-launch kernel beats the bucket + pack chain, and uses that crossover from then on (the built-in values were
 * measured on one GPU).  The live inventory is preserved.  *crossover_claims (may be NULL) receives the result. */
int  dra_calibrate(dra_ctx* ctx, uint32_t* crossover_claims);

/* ---- resident mode (DRA_CFG_RESIDENT) ------------------------------------------------------------------------------
 * Optional explicit control: start the resident kernel now (the first eligible dra_allocate_batch would), stop it (every
 * other entry point of the context does so implicitly before it runs).  dra_serve_batches: batches it has answered. */
int  dra_serve_start(dra_ctx* ctx);
int  dra_serve_stop(dra_ctx* ctx);
uint64_t dra_serve_batches(const dra_ctx* ctx);

/* ---- host memory + instrumentation ---------------------------------------------------------------- */

/* Page-locked host buffers: passing these to the *_batch calls skips the internal staging copy. */
void* dra_host_alloc(size_t bytes);
void  dra_host_free(void* p);

/* Kernel launches issued by this context since creation (all of them this library's own kernels). */
uint64_t dra_launch_count(const dra_ctx* ctx);
/* When enabled, CUDA events bracket each kernel of the next calls; dra_get_timings returns the last
 * call's per-stage device times in microseconds: [0] bucket-hist [1] bucket-scan [2] bucket-scatter
 * [3] pack [4] all-gather.  Returns the number of floats written. */
int  dra_set_profiling(dra_ctx* ctx, int enabled);
/* Instrumentation (env DRA_TIMELINE=1): 8 clock stamps per CTA of the last single-launch kernel; returns the
 * number of u64 words copied to host. */
int  dra_debug_timeline(dra_ctx* ctx, unsigned long long* host, uint32_t n);
/* Kernels enqueued by the last Allocate-family call on this context (DRA_K_* bits) and the hist tile it used (claims per
 * tile of k_bucket_hist8 / k_bucket_hist; 0 when the call ran neither).  A CUDA-graph replay reports the chain of the call
 * that was captured.  Returns DRA_OK. */
int  dra_debug_last_chain(const dra_ctx* ctx, uint32_t* kernels, uint32_t* hist_tile);
#define DRA_K_FUSED_STAGED      0x00001u  /* single-launch kernel, claim array staged in shared memory */
#define DRA_K_FUSED_STREAM      0x00002u  /* single-launch kernel, claims streamed from global memory */
#define DRA_K_FUSED_DIRECT      0x00004u  /* single-launch kernel reading / writing the pinned host buffers (cooperative) */
#define DRA_K_SERVE             0x00008u  /* the batch was answered by the resident kernel */
#define DRA_K_SORTED_PREP       0x00010u  /* DRA_F_NODE_SORTED: k_sorted_prep instead of the counting sort */
#define DRA_K_BUCKET_SMALL      0x00020u  /* the whole counting sort in one CTA */
#define DRA_K_HIST8             0x00040u  /* CTA-wide histogram, 2048-claim tiles */
#define DRA_K_HIST8_MULTI       0x00080u  /* CTA-wide histogram, tiles grown to a multiple of 2048 */
#define DRA_K_HIST_WARP         0x00100u  /* one-warp histogram tiles (node ranges too wide for the CTA-wide form) */
#define DRA_K_SCAN8             0x00200u  /* scan of the tile histograms: one warp per node */
#define DRA_K_SCAN_ROWS         0x00400u  /* scan of the tile histograms: coalesced rows, look-back over CTAs */
#define DRA_K_SCAN              0x00800u  /* scan of the one-warp histograms: one CTA */
#define DRA_K_SCATTER           0x01000u
#define DRA_K_PACK1             0x02000u  /* one warp per node, one node per CTA */
#define DRA_K_PACK4             0x04000u  /* CTAs of four warps, each warp walking several nodes */
#define DRA_K_COMPACT_FLAT1     0x08000u  /* sharded call: compaction in 256-claim tiles */
#define DRA_K_COMPACT_FLAT8     0x10000u  /* sharded call: compaction in 2048-claim tiles */
#define DRA_K_COMPACT_LOOKBACK  0x20000u  /* sharded call: compaction with a decoupled look-back (beyond 2M claims) */
#define DRA_K_COMPACT_IN_KERNEL 0x40000u  /* sharded call: compaction inside the single-launch kernel */
#define DRA_K_POD_SHARD         0x80000u  /* sharded pods Allocate: pod records + ownership, gate, k_pods on the node window */
#define DRA_K_POD_GATHER        0x100000u /* sharded pods Allocate: all-gather of the owned pods' records (world > 1) */
#define DRA_K_PLACE             0x200000u /* place pods: pod states + pair records, persistent walk of the nodes' visit lists */
#define DRA_K_PLACE_SHARD       0x400000u /* sharded place pods: prep, gate, walk of the node window, finalisers (+ all-gather) */
#define DRA_K_PREEMPT           0x800000u /* preemption: running-pod prep, victim lists, pairs, choice, victim rows */
#define DRA_K_PREEMPT_SHARD    0x1000000u /* sharded preemption: prep, victim lists, the window's pairs, partials, merge */
#define DRA_K_PREEMPT_PLACE    0x2000000u /* preempt and place: running-pod prep, victim lists, visit lists, persistent walk */
#define DRA_K_PREEMPT_PLACE_SHARD 0x4000000u /* sharded preempt and place: state exchange, the §15 chain on it, own range back */
#define DRA_K_POD_CAPACITY     0x8000000u /* pod capacity: the pairs' copy counts, the per-pod sums */
#define DRA_K_POD_CAPACITY_SHARD 0x10000000u /* sharded pod capacity: prep, the window's pairs, exchange, merge with the sums */
/* Instrumentation (env DRA_TIMELINE=1): globaltimer of the last shard compaction's first CTA in / last CTA out. */
int  dra_debug_shard_times(dra_ctx* ctx, unsigned long long* two);
/* Instrumentation: globaltimer stamps of the resident kernel's last batch — doorbell seen, CTA 0's egress issued, every CTA
 * fenced, completion word written.  Stops the resident kernel. */
int  dra_debug_serve_times(dra_ctx* ctx, unsigned long long* four);
/* Instrumentation: enqueue an empty kernel of the given shape on ctx's stream (launch-floor calibration). */
int  dra_debug_noop(dra_ctx* ctx, uint32_t grid, uint32_t block, uint32_t smem_bytes);
int  dra_get_timings(dra_ctx* ctx, float* us, int n);

#ifdef __cplusplus
}
#endif
#endif /* DRA_ALLOC_H */
