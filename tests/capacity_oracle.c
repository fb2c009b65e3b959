/*
 * capacity_oracle.c — CPU oracle of spec §16 (pod capacity).  TEST INFRASTRUCTURE ONLY, built by tests/capacity_oracle.py.
 *
 * Every evaluation is the §12 pod evaluation of oracle/dra_oracle.c itself (its static pod_eval, included below), on a
 * private copy of the node that keeps each placement that succeeds.  Restated here: the counting loop, the reason it
 * stopped and the per-pod sums.
 */
#include "../oracle/dra_oracle.c"

#define CAPACITY_API __attribute__((visibility("default")))

CAPACITY_API void capacity_oracle_set_selectors(const dra_gpu_attr* attrs, uint32_t n_gpu, const dra_selector* sels, uint32_t n_sel)
{
    dra_oracle_set_selectors(attrs, n_gpu, sels, n_sel);
}

/* Returns -1, with nothing written, on the arguments spec §16 rejects.  pair_stop, pod_total and pod_nodes may be NULL. */
CAPACITY_API int capacity_oracle_capacity(const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                                          const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                                          const uint32_t* pod_off, uint32_t n_pod,
                                          const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t max_copies,
                                          uint16_t* pair_copies, uint8_t* pair_stop, uint64_t* pod_total, uint32_t* pod_nodes,
                                          uint32_t flags)
{
    if (flags & ~(uint32_t)DRA_F_EXHAUSTIVE) return -1;
    if (max_copies < 1 || max_copies > 65535) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (pod_off[0] != 0 || pod_off[n_pod] != n_claim) return -1;
    for (uint32_t p = 0; p < n_pod; p++) if (pod_off[p + 1] < pod_off[p]) return -1;
    const int dense = cand_nodes == NULL && cand_off == NULL;
    if (!dense) {
        if (!cand_off || cand_off[0] != 0) return -1;
        for (uint32_t p = 0; p < n_pod; p++) if (cand_off[p + 1] < cand_off[p]) return -1;
        if (cand_off[n_pod] && !cand_nodes) return -1;
    } else if ((uint64_t)n_pod * n_node >= (1ull << 32)) return -1;
    if ((dense ? (uint64_t)n_pod * n_node : cand_off[n_pod]) && !pair_copies) return -1;

    const int exh = (flags & DRA_F_EXHAUSTIVE) != 0;
    dra_claim_rec pod[DRA_MAX_POD];
    dra_gpu_rec S[DRA_MAX_GPUS_PER_NODE];
    dra_out_rec o[DRA_MAX_POD * DRA_MAX_COUNT];
    uint32_t slot[DRA_MAX_POD];
    for (uint32_t p = 0; p < n_pod; p++) {
        uint32_t c0 = pod_off[p], cnt = pod_off[p + 1] - c0;
        uint32_t k0 = dense ? (uint32_t)((uint64_t)p * n_node) : cand_off[p];
        uint32_t k1 = dense ? (uint32_t)((uint64_t)p * n_node + n_node) : cand_off[p + 1];
        uint64_t total = 0; uint32_t nodes = 0;
        for (uint32_t k = k0; k < k1; k++) {
            uint32_t n = dense ? k - k0 : cand_nodes[k];
            uint32_t copies = 0; uint8_t stop = DRA_ST_POD;
            if (n >= n_node) { /* no such node: unsuitable */ }
            else if (cnt == 0) { copies = max_copies; stop = DRA_ST_OK; }
            else if (cnt > DRA_MAX_POD) stop = DRA_ST_INVALID;
            else {
                uint32_t g0 = node_off[n], ng = node_off[n + 1] - g0, t = 0;
                int inv = 0;
                for (uint32_t i = 0; i < cnt; i++) {
                    pod[i] = claims[c0 + i]; pod[i].node = n;
                    slot[i] = t; t += claim_slots(&pod[i], n_node, 1);
                    inv = inv || claim_invalid(&pod[i], n_node, 1);
                }
                memcpy(S, gpus + g0, ng * sizeof *S);
                stop = DRA_ST_OK;
                while (copies < max_copies) {
                    if (!pod_eval(S, g0, ng, tbl, pod, cnt, n_node, 1, slot, o, exh)) {
                        stop = inv ? DRA_ST_INVALID : o[0].status == DRA_ST_SEARCH_LIMIT ? DRA_ST_SEARCH_LIMIT : DRA_ST_POD;
                        break;
                    }
                    copies++;
                }
            }
            pair_copies[k] = (uint16_t)copies;
            if (pair_stop) pair_stop[k] = stop;
            total += copies; nodes += copies != 0;
        }
        if (pod_total) pod_total[p] = total;
        if (pod_nodes) pod_nodes[p] = nodes;
    }
    return 0;
}
