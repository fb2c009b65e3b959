/*
 * dra_oracle.h — CPU oracle of spec/ALLOCATION.md.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this.
 * The product (libdra_alloc.so) never links, loads or calls it.
 *
 * PARITY UNPINNED for the search itself: the reference snapshot has no Allocate()/UnsuitableNodes()
 * implementation and no test of one (SURVEY.md F1, F5), and Go is absent from this image.  What the
 * snapshot does pin is restated with file:line citations in dra_oracle.c and checked against the
 * reference's own vectors: the MPS limit table of sharing_test.go:37-149 and the gpu-test4 geometry.
 */
#ifndef DRA_ORACLE_H
#define DRA_ORACLE_H

#include "../include/dra_alloc.h"   /* record layouts only */

#ifdef __cplusplus
extern "C" {
#endif

/* Allocate batch (spec §2-§7).  Mutates gpus[].  Returns 0, or -1 on malformed arguments
 * (out_off[i]+slots > n_out, node_off not monotone, > 32 GPUs in a node). */
int dra_oracle_allocate(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                        const dra_profile_tbl* tbl /* [DRA_MAX_MODELS] */,
                        const dra_claim_rec* claims, uint32_t n_claim,
                        const uint32_t* out_off, dra_out_rec* out, uint32_t n_out);

/* Same result, nodes processed by n_threads threads: the caller plus a persistent pool of n_threads-1 workers that
 * take nodes one at a time (nodes are independent, spec §2).  The pool is created on first use and resized when
 * n_threads changes; one call at a time. */
int dra_oracle_allocate_mt(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                           const dra_profile_tbl* tbl,
                           const dra_claim_rec* claims, uint32_t n_claim,
                           const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, int n_threads);

/* Optional selector context for the calls that follow (spec §10); pass NULL / 0 to clear.  Not thread-safe
 * with respect to concurrent calls (test infrastructure). */
void dra_oracle_set_selectors(const dra_gpu_attr* attrs, uint32_t n_gpu, const dra_selector* sels, uint32_t n_sel);

/* UnsuitableNodes (spec §8).  gpus is read-only. */
int dra_oracle_unsuitable(const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off,
                          uint32_t n_node, const dra_profile_tbl* tbl,
                          const dra_claim_rec* claims, uint32_t n_claim,
                          const uint32_t* pod_off, uint32_t n_pod,
                          const uint32_t* cand_nodes, const uint32_t* cand_off, uint8_t* suitable_bits);

/* Pod mode (spec §12): Allocate with pod boundaries, atomic per pod; flags & DRA_F_EXHAUSTIVE = backtracking search. */
int dra_oracle_allocate_pods(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                             const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                             const uint32_t* pod_off, uint32_t n_pod,
                             const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, uint32_t flags);
/* UnsuitableNodes with flags (DRA_F_EXHAUSTIVE: spec §12; 0: spec §8, same as dra_oracle_unsuitable). */
int dra_oracle_unsuitable_ex(const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off,
                             uint32_t n_node, const dra_profile_tbl* tbl,
                             const dra_claim_rec* claims, uint32_t n_claim,
                             const uint32_t* pod_off, uint32_t n_pod,
                             const uint32_t* cand_nodes, const uint32_t* cand_off, uint8_t* suitable_bits,
                             uint32_t flags);

/* Deallocate (spec §9).  -1, with gpus untouched, when a claim's slot range leaves [0, n_out). */
int dra_oracle_deallocate(dra_gpu_rec* gpus, uint32_t n_gpu, uint32_t n_node,
                          const dra_claim_rec* claims, uint32_t n_claim,
                          const uint32_t* out_off, const dra_out_rec* out, uint32_t n_out);

/* limit.Megabyte(): api/nvidia.com/resource/gpu/v1alpha1/sharing.go:234-237 —
 * v = bytes/1024/1024 (Go integer division, truncation toward zero), valid iff v > 0. */
int64_t dra_oracle_megabyte(int64_t bytes, int* valid);

/* imexDomainOffsets.add's search: cmd/nvidia-dra-controller/imex.go:336-349 — lowest multiple of
 * `step` below `limit` not present in used[0..n_used); -1 when none ("channel limit reached"). */
int32_t dra_oracle_imex_offset(const int32_t* used, uint32_t n_used, int32_t step, int32_t limit);

#ifdef __cplusplus
}
#endif
#endif
