/*
 * preempt_place_oracle.c — CPU oracle of spec §15 (preempt and place).  TEST INFRASTRUCTURE ONLY, built by
 * tests/preempt_place_oracle.py.
 *
 * The pair judgement, the victim order and the choice are tests/preempt_oracle.c's (included below, and through it the §12
 * pod evaluation of oracle/dra_oracle.c).  Restated here: the sequential schedule.  Pods in input order, each judged on
 * the CURRENT inventory against the running pods not evicted yet, then applied: §9 for the victims, §12 on the chosen node.
 */
#include "preempt_oracle.c"

PREEMPT_API void pp_oracle_set_selectors(const dra_gpu_attr* attrs, uint32_t n_gpu, const dra_selector* sels, uint32_t n_sel)
{
    dra_oracle_set_selectors(attrs, n_gpu, sels, n_sel);
}

/* Mutates gpus[].  cand_nodes == cand_off == NULL: every node, ascending.  Returns -1, with nothing written and gpus[]
 * unchanged, on the arguments spec §15 rejects. */
PREEMPT_API int pp_oracle_preempt_place(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                                        const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                                        const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                                        const uint32_t* cand_nodes, const uint32_t* cand_off,
                                        const dra_claim_rec* rclaims, uint32_t rn_claim, const uint32_t* rpod_off,
                                        const int32_t* rprio, uint32_t rn_pod, const uint32_t* rout_off,
                                        const dra_out_rec* rout, uint32_t rn_out,
                                        const uint32_t* out_off, dra_out_rec* out, uint32_t n_out,
                                        uint32_t* pod_node, uint8_t* pod_status, uint32_t* evicted_by, uint32_t flags)
{
    const uint32_t POS_MAX = 0x3FFFFFFFu;
    if (flags & ~(uint32_t)DRA_F_EXHAUSTIVE) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (n_node > POS_MAX) return -1;
    if (pod_off[0] != 0 || pod_off[n_pod] != n_claim) return -1;
    for (uint32_t p = 0; p < n_pod; p++) if (pod_off[p + 1] < pod_off[p]) return -1;
    const int dense = cand_nodes == NULL && cand_off == NULL;
    if (!dense) {
        if (!cand_off || cand_off[0] != 0) return -1;
        for (uint32_t p = 0; p < n_pod; p++)
            if (cand_off[p + 1] < cand_off[p] || cand_off[p + 1] - cand_off[p] > POS_MAX) return -1;
    } else if ((uint64_t)n_pod * n_node >= (1ull << 32)) return -1;
    const int have_off = out_off != NULL;
    for (uint32_t i = 0; i < n_claim; i++) {              /* slots as if the claim named a node of the inventory */
        dra_claim_rec t = claims[i]; t.node = 0;
        uint32_t b = have_off ? out_off[i] : i, sl = claim_slots(&t, 1, have_off);
        if (b > n_out || sl > n_out - b) return -1;
    }
    if (n_pod == 0) return 0;                             /* no pending pods: the running pods are not examined */
    if (rpod_off[0] != 0 || rpod_off[rn_pod] != rn_claim) return -1;
    for (uint32_t r = 0; r < rn_pod; r++) if (rpod_off[r + 1] < rpod_off[r]) return -1;
    running R = { rclaims, rpod_off, rprio, rout_off, rout, n_node };
    uint32_t* rnode = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    if (!rnode) return -1;
    for (uint32_t r = 0; r < rn_pod; r++) {
        rnode[r] = DRA_GPU_NONE;
        for (uint32_t i = rpod_off[r]; i < rpod_off[r + 1]; i++) {
            uint32_t base = rout_off ? rout_off[i] : i, sl = run_slots(&rclaims[i], n_node, rout_off != NULL);
            if (base > rn_out || sl > rn_out - base) { free(rnode); return -1; }
            for (uint32_t k = 0; k < sl; k++) {
                const dra_out_rec* o = &rout[base + k];
                if (o->status != DRA_ST_OK) continue;
                if (o->gpu >= n_gpu) { free(rnode); return -1; }
                uint32_t n = gpus[o->gpu].node;
                if (rnode[r] == DRA_GPU_NONE) rnode[r] = n;
                else if (rnode[r] != n) { free(rnode); return -1; }
            }
        }
    }
    /* per node: its running pods not evicted yet, by priority descending, then index: list[loff[n] .. lend[n]) */
    uint32_t* loff = (uint32_t*)calloc((size_t)n_node + 2, sizeof(uint32_t));
    uint32_t* lend = (uint32_t*)calloc((size_t)n_node + 1, sizeof(uint32_t));
    uint32_t* list = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    uint32_t* vic = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    if (!loff || !lend || !list || !vic) { free(rnode); free(loff); free(lend); free(list); free(vic); return -1; }
    for (uint32_t r = 0; r < rn_pod; r++) if (rnode[r] < n_node) loff[rnode[r] + 1]++;
    for (uint32_t n = 0; n < n_node; n++) loff[n + 1] += loff[n];
    for (uint32_t r = 0; r < rn_pod; r++) if (rnode[r] < n_node) list[loff[rnode[r]]++] = r;
    for (uint32_t n = n_node; n > 0; n--) loff[n] = loff[n - 1];
    loff[0] = 0;
    g_rprio = rprio;
    for (uint32_t n = 0; n < n_node; n++) {
        qsort(list + loff[n], loff[n + 1] - loff[n], sizeof(uint32_t), by_prio_desc);
        lend[n] = loff[n + 1];
    }
    for (uint32_t r = 0; r < rn_pod; r++) evicted_by[r] = DRA_GPU_NONE;

    const int exh = (flags & DRA_F_EXHAUSTIVE) != 0;
    dra_claim_rec pod[DRA_MAX_POD];
    for (uint32_t p = 0; p < n_pod; p++) {
        uint32_t c0 = pod_off[p], cnt = pod_off[p + 1] - c0;
        uint32_t k0 = dense ? 0 : cand_off[p], k1 = dense ? n_node : cand_off[p + 1];
        int have_best = 0, any_lim = 0; uint32_t fit_k = DRA_GPU_NONE, best_k = 0;
        pair_sum best = { 0 };
        for (uint32_t k = k0; k < k1; k++) {              /* §14's pairs on the current state */
            uint32_t n = dense ? k : cand_nodes[k];
            if (n < n_node && cnt <= DRA_MAX_POD)
                for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, n < n_node ? loff[n] : 0,
                               n < n_node ? lend[n] : 0, exh, NULL);
            if (s.st == PRE_FITS && fit_k == DRA_GPU_NONE) fit_k = k;
            if (s.st == PRE_LIMIT) any_lim = 1;
            if (s.st == PRE_EVICT && (!have_best || better(&s, &best))) { best = s; best_k = k; have_best = 1; }
        }
        uint32_t n = DRA_GPU_NONE;
        if (fit_k != DRA_GPU_NONE) { n = dense ? fit_k : cand_nodes[fit_k]; pod_status[p] = PRE_FITS; }
        else if (have_best) { n = dense ? best_k : cand_nodes[best_k]; pod_status[p] = PRE_EVICT; }
        else {
            int inv = cnt > DRA_MAX_POD;
            for (uint32_t i = 0; i < cnt && !inv; i++) { dra_claim_rec t = claims[c0 + i]; t.node = 0; inv = claim_invalid(&t, 1, 1); }
            pod_status[p] = inv ? PRE_INVALID : any_lim ? PRE_LIMIT : PRE_NO;
        }
        pod_node[p] = n;
        if (n == DRA_GPU_NONE) {                          /* placed nowhere: the inventory is unchanged */
            for (uint32_t i = c0; i < c0 + cnt; i++) {
                dra_claim_rec t = claims[i]; t.node = 0;
                int inv = cnt > DRA_MAX_POD || claim_invalid(&t, 1, have_off);
                fail_all(&out[have_off ? out_off[i] : i], claim_slots(&t, 1, have_off), &t,
                         inv ? DRA_ST_INVALID : pod_status[p] == PRE_LIMIT ? DRA_ST_SEARCH_LIMIT : DRA_ST_POD);
            }
            continue;
        }
        uint32_t g0 = node_off[n], ng = node_off[n + 1] - g0;
        for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
        if (pod_status[p] == PRE_EVICT) {                 /* §9 for the victims, gone from the node's list */
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, loff[n], lend[n], exh, vic);
            for (uint32_t j = 0; j < s.count; j++) { run_apply(&R, vic[j], gpus + g0, g0, ng, 0); evicted_by[vic[j]] = p; }
            uint32_t w = loff[n];
            for (uint32_t v = loff[n]; v < lend[n]; v++) if (evicted_by[list[v]] == DRA_GPU_NONE) list[w++] = list[v];
            lend[n] = w;
        }
        if (cnt == 0) continue;                           /* an empty pod: nothing to write */
        uint32_t slot[DRA_MAX_POD];
        for (uint32_t i = 0; i < cnt; i++) slot[i] = have_off ? out_off[c0 + i] : c0 + i;
        (void)pod_eval(gpus + g0, g0, ng, tbl, pod, cnt, n_node, have_off, slot, out, exh);   /* §12 on the chosen node */
    }
    free(rnode); free(loff); free(lend); free(list); free(vic);
    return 0;
}
