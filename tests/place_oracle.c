/*
 * place_oracle.c — CPU oracle of spec §13 (place pods).  TEST INFRASTRUCTURE ONLY, built by tests/place_oracle.py.
 *
 * The sequential rule, literally: pods in input order, each on its candidates in list order, every evaluation on the
 * candidate's CURRENT state (the classic controller's pending allocations, SURVEY App. A).  Each evaluation is the §12
 * pod evaluation of oracle/dra_oracle.c itself (its static pod_eval, included below), so the only thing restated here is
 * the walk over candidates.
 */
#include "../oracle/dra_oracle.c"

#define PLACE_API __attribute__((visibility("default")))

PLACE_API void place_oracle_set_selectors(const dra_gpu_attr* attrs, uint32_t n_gpu, const dra_selector* sels, uint32_t n_sel)
{
    dra_oracle_set_selectors(attrs, n_gpu, sels, n_sel);
}

/* Mutates gpus[]; pod_node[p] = the node pod p was placed on, or 0xFFFFFFFF.  cand_nodes == cand_off == NULL: every node,
 * ascending.  flags: DRA_F_EXHAUSTIVE (DRA_F_FRESH_INVENTORY is accepted and has no effect: gpus[] is the starting
 * state).  Returns -1, with nothing changed, on the arguments spec §13 rejects. */
PLACE_API int place_oracle_place_pods(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                                      const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                                      const uint32_t* pod_off, uint32_t n_pod,
                                      const uint32_t* cand_nodes, const uint32_t* cand_off,
                                      const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, uint32_t* pod_node,
                                      uint32_t flags)
{
    if (flags & ~(uint32_t)(DRA_F_EXHAUSTIVE | DRA_F_FRESH_INVENTORY)) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (pod_off[0] != 0 || pod_off[n_pod] != n_claim) return -1;
    for (uint32_t p = 0; p < n_pod; p++) if (pod_off[p + 1] < pod_off[p]) return -1;
    const int dense = cand_nodes == NULL && cand_off == NULL;
    if (!dense) {
        if (!cand_off || cand_off[0] != 0) return -1;
        for (uint32_t p = 0; p < n_pod; p++) if (cand_off[p + 1] < cand_off[p]) return -1;
    }
    int have_off = out_off != NULL;
    /* slots as if every claim named a node of the inventory: the node it ends on is not known up front */
    uint32_t* slot = (uint32_t*)malloc(((size_t)n_claim + 1) * sizeof(uint32_t));
    if (!slot) return -1;
    for (uint32_t i = 0; i < n_claim; i++) {
        dra_claim_rec t = claims[i]; t.node = 0;
        slot[i] = have_off ? out_off[i] : i;
        uint32_t sl = claim_slots(&t, 1, have_off);
        if (slot[i] > n_out || sl > n_out - slot[i]) { free(slot); return -1; }
    }
    dra_claim_rec pod[DRA_MAX_POD];
    for (uint32_t p = 0; p < n_pod; p++) {
        uint32_t c0 = pod_off[p], cnt = pod_off[p + 1] - pod_off[p];
        pod_node[p] = DRA_GPU_NONE;
        if (cnt == 0) continue;
        if (cnt > DRA_MAX_POD) {
            for (uint32_t i = c0; i < c0 + cnt; i++) {
                dra_claim_rec t = claims[i]; t.node = 0;
                fail_all(&out[slot[i]], claim_slots(&t, 1, have_off), &t, DRA_ST_INVALID);
            }
            continue;
        }
        uint32_t k0 = dense ? 0 : cand_off[p], k1 = dense ? n_node : cand_off[p + 1];
        int limit = 0;
        for (uint32_t k = k0; k < k1 && pod_node[p] == DRA_GPU_NONE; k++) {
            uint32_t n = dense ? k : cand_nodes[k];
            if (n >= n_node) continue;                       /* names no node of the inventory: skipped */
            for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
            if (pod_eval(gpus + node_off[n], node_off[n], node_off[n + 1] - node_off[n], tbl, pod, cnt, n_node,
                         have_off, slot + c0, out, (flags & DRA_F_EXHAUSTIVE) != 0))
                pod_node[p] = n;
            else if (out[slot[c0]].status == DRA_ST_SEARCH_LIMIT)   /* (an INVALID claim fails the pod before any search) */
                limit = 1;
        }
        if (pod_node[p] != DRA_GPU_NONE) continue;
        for (uint32_t i = 0; i < cnt; i++) {                 /* placed nowhere (or no usable candidate at all) */
            dra_claim_rec t = claims[c0 + i]; t.node = 0;
            int inv = claim_invalid(&t, 1, have_off);
            fail_all(&out[slot[c0 + i]], claim_slots(&t, 1, have_off), &t,
                     inv ? DRA_ST_INVALID : limit ? DRA_ST_SEARCH_LIMIT : DRA_ST_POD);
        }
    }
    free(slot);
    return 0;
}
