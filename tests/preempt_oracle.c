/*
 * preempt_oracle.c — CPU oracle of spec §14 (preemption).  TEST INFRASTRUCTURE ONLY, built by tests/preempt_oracle.py.
 *
 * Every evaluation is the §12 pod evaluation of oracle/dra_oracle.c itself (its static pod_eval, included below), on a
 * private copy of the node.  Restated here: the §9 update of a running pod and its inverse, the victim ordering, the
 * reprieve and the choice of the node.
 */
#include "../oracle/dra_oracle.c"

#define PREEMPT_API __attribute__((visibility("default")))

enum { PRE_FITS = 0, PRE_EVICT = 1, PRE_NO = 2, PRE_LIMIT = 3, PRE_INVALID = 4 };

PREEMPT_API void preempt_oracle_set_selectors(const dra_gpu_attr* attrs, uint32_t n_gpu, const dra_selector* sels, uint32_t n_sel)
{
    dra_oracle_set_selectors(attrs, n_gpu, sels, n_sel);
}

typedef struct running {
    const dra_claim_rec* claims; const uint32_t* pod_off; const int32_t* prio;
    const uint32_t* out_off; const dra_out_rec* out; uint32_t n_node;
} running;

/* slots(c) as §9 counts them: the claim's own node field decides, as it did for Allocate */
static uint32_t run_slots(const dra_claim_rec* c, uint32_t n_node, int have_off)
{
    return (c->kind == DRA_KIND_GPU && c->node < n_node && c->count >= 1 && c->count <= DRA_MAX_COUNT &&
            (have_off || c->count == 1)) ? c->count : 1u;
}

static uint16_t slice_mask(uint8_t start, uint8_t size)
{
    uint32_t m = size >= 16 ? 0xFFFFu : (1u << size) - 1u;
    return start >= 16 ? 0 : (uint16_t)(m << start);
}

/* running pod r's OK slots applied to the node's GPUs gpus[0..ng) (global index g0..): add = the Allocate updates,
 * otherwise the §9 inverse; u16 / u32 wrap-around as the records hold them */
static void run_apply(const running* R, uint32_t r, dra_gpu_rec* gpus, uint32_t g0, uint32_t ng, int add)
{
    for (uint32_t i = R->pod_off[r]; i < R->pod_off[r + 1]; i++) {
        const dra_claim_rec* c = &R->claims[i];
        uint32_t base = R->out_off ? R->out_off[i] : i, sl = run_slots(c, R->n_node, R->out_off != NULL);
        for (uint32_t k = 0; k < sl; k++) {
            const dra_out_rec* o = &R->out[base + k];
            if (o->status != DRA_ST_OK || o->gpu < g0 || o->gpu - g0 >= ng) continue;
            dra_gpu_rec* g = &gpus[o->gpu - g0];
            if (c->kind == DRA_KIND_GPU) {
                if (add) g->flags |= DRA_GPU_FULL_ALLOCATED; else g->flags &= (uint8_t)~DRA_GPU_FULL_ALLOCATED;
            } else if (c->kind == DRA_KIND_MIG) {
                uint16_t m = slice_mask(o->start, o->size);
                if (add) g->busy |= m; else g->busy &= (uint16_t)~m;
            } else if (c->kind == DRA_KIND_SHARED) {
                if (add) { g->mem_free_mib -= c->mem_limit_mib; g->share_cnt++; }
                else { g->mem_free_mib += c->mem_limit_mib; g->share_cnt--; }
            }
        }
    }
}

/* 1 placed, 0 not; *lim set on SEARCH_LIMIT */
static int eval_on(const dra_gpu_rec* S, uint32_t g0, uint32_t ng, const dra_profile_tbl* tbl, const dra_claim_rec* pod,
                   uint32_t cnt, uint32_t n_node, int exh, int* lim)
{
    dra_gpu_rec w[DRA_MAX_GPUS_PER_NODE];
    dra_out_rec o[DRA_MAX_POD * DRA_MAX_COUNT];
    uint32_t slot[DRA_MAX_POD] = { 0 }, t = 0;
    for (uint32_t i = 0; i < cnt; i++) { slot[i] = t; t += claim_slots(&pod[i], n_node, 1); }
    memcpy(w, S, ng * sizeof *w);
    if (pod_eval(w, g0, ng, tbl, pod, cnt, n_node, 1, slot, o, exh)) return 1;
    *lim = cnt > 0 && o[0].status == DRA_ST_SEARCH_LIMIT;
    return 0;
}

typedef struct pair_sum {
    uint8_t st; uint32_t count; int32_t hi; uint64_t sum; uint32_t hi_idx;
} pair_sum;

static const int32_t* g_rprio;     /* qsort has no context argument */
static int by_prio_desc(const void* a, const void* b)
{
    uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
    if (g_rprio[x] != g_rprio[y]) return g_rprio[x] > g_rprio[y] ? -1 : 1;
    return x < y ? -1 : x > y;
}

/* Pair (pod, node n): writes the victims (running-pod indices, V order) into vic when non-NULL */
static pair_sum judge(const dra_gpu_rec* gpus, const uint32_t* node_off, uint32_t n_node, const dra_profile_tbl* tbl,
                      const dra_claim_rec* pod, uint32_t cnt, int32_t prio, uint32_t n, const running* R,
                      const uint32_t* list, uint32_t l0, uint32_t l1, int exh, uint32_t* vic)
{
    pair_sum s = { PRE_NO, 0, INT32_MIN, 0, 0xFFFFFFFFu };
    if (n >= n_node) return s;
    if (cnt > DRA_MAX_POD) { s.st = PRE_INVALID; return s; }
    uint32_t g0 = node_off[n], ng = node_off[n + 1] - g0;
    int lim = 0;
    if (eval_on(gpus + g0, g0, ng, tbl, pod, cnt, n_node, exh, &lim)) { s.st = PRE_FITS; return s; }
    for (uint32_t i = 0; i < cnt; i++) if (claim_invalid(&pod[i], n_node, 1)) { s.st = PRE_INVALID; return s; }
    dra_gpu_rec S[DRA_MAX_GPUS_PER_NODE], S2[DRA_MAX_GPUS_PER_NODE];
    memcpy(S, gpus + g0, ng * sizeof *S);
    uint32_t v0 = l0;                                    /* V = list[v0 .. l1): priority strictly below the pod's */
    while (v0 < l1 && R->prio[list[v0]] >= prio) v0++;
    for (uint32_t v = v0; v < l1; v++) run_apply(R, list[v], S, g0, ng, 0);
    lim = 0;
    if (!eval_on(S, g0, ng, tbl, pod, cnt, n_node, exh, &lim)) { s.st = lim ? PRE_LIMIT : PRE_NO; return s; }
    s.st = PRE_EVICT;
    for (uint32_t v = v0; v < l1; v++) {
        uint32_t r = list[v];
        memcpy(S2, S, ng * sizeof *S);
        run_apply(R, r, S2, g0, ng, 1);
        if (eval_on(S2, g0, ng, tbl, pod, cnt, n_node, exh, &lim)) { memcpy(S, S2, ng * sizeof *S); continue; }
        if (s.count == 0) { s.hi = R->prio[r]; s.hi_idx = r; }     /* V order: the first victim has the highest priority */
        s.sum += (uint64_t)((int64_t)R->prio[r] + 2147483648ll);
        if (vic) vic[s.count] = r;
        s.count++;
    }
    return s;
}

/* 1 when a is preferred to b (pickOneNodeForPreemption without start times and PDBs) */
static int better(const pair_sum* a, const pair_sum* b)
{
    if (a->hi != b->hi) return a->hi < b->hi;
    if (a->sum != b->sum) return a->sum < b->sum;
    if (a->count != b->count) return a->count < b->count;
    if (a->hi_idx != b->hi_idx) return a->hi_idx > b->hi_idx;
    return 0;                                            /* equal: the earlier candidate stays */
}

/* Returns -1, with nothing written, on the arguments spec §14 rejects. */
PREEMPT_API int preempt_oracle_preempt(const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                                       const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                                       const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                                       const uint32_t* cand_nodes, const uint32_t* cand_off,
                                       const dra_claim_rec* rclaims, uint32_t rn_claim, const uint32_t* rpod_off,
                                       const int32_t* rprio, uint32_t rn_pod, const uint32_t* rout_off,
                                       const dra_out_rec* rout, uint32_t rn_out,
                                       uint8_t* pair_status, uint32_t* pair_victims, uint32_t* pod_node, uint8_t* pod_status,
                                       uint32_t* n_victims, uint32_t* victims, uint32_t max_victims, uint32_t flags)
{
    if (flags & ~(uint32_t)DRA_F_EXHAUSTIVE) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (pod_off[0] != 0 || pod_off[n_pod] != n_claim) return -1;
    for (uint32_t p = 0; p < n_pod; p++) if (pod_off[p + 1] < pod_off[p]) return -1;
    const int dense = cand_nodes == NULL && cand_off == NULL;
    if (!dense) {
        if (!cand_off || cand_off[0] != 0) return -1;
        for (uint32_t p = 0; p < n_pod; p++) if (cand_off[p + 1] < cand_off[p]) return -1;
    } else if ((uint64_t)n_pod * n_node >= (1ull << 32)) return -1;
    if (rpod_off[0] != 0 || rpod_off[rn_pod] != rn_claim) return -1;
    for (uint32_t r = 0; r < rn_pod; r++) if (rpod_off[r + 1] < rpod_off[r]) return -1;
    if (max_victims && !victims) return -1;
    running R = { rclaims, rpod_off, rprio, rout_off, rout, n_node };
    /* where each running pod is: the node of its OK slots' GPUs */
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
    /* per node: its running pods by priority descending, then index */
    uint32_t* loff = (uint32_t*)calloc((size_t)n_node + 2, sizeof(uint32_t));
    uint32_t* list = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    uint32_t* vic = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    if (!loff || !list || !vic) { free(rnode); free(loff); free(list); free(vic); return -1; }
    for (uint32_t r = 0; r < rn_pod; r++) if (rnode[r] < n_node) loff[rnode[r] + 1]++;
    for (uint32_t n = 0; n < n_node; n++) loff[n + 1] += loff[n];
    for (uint32_t r = 0; r < rn_pod; r++) if (rnode[r] < n_node) list[loff[rnode[r]]++] = r;
    for (uint32_t n = n_node; n > 0; n--) loff[n] = loff[n - 1];
    loff[0] = 0;
    g_rprio = rprio;
    for (uint32_t n = 0; n < n_node; n++) qsort(list + loff[n], loff[n + 1] - loff[n], sizeof(uint32_t), by_prio_desc);

    const int exh = (flags & DRA_F_EXHAUSTIVE) != 0;
    dra_claim_rec pod[DRA_MAX_POD];
    for (uint32_t p = 0; p < n_pod; p++) {
        uint32_t c0 = pod_off[p], cnt = pod_off[p + 1] - c0;
        uint32_t k0 = dense ? (uint32_t)((uint64_t)p * n_node) : cand_off[p];
        uint32_t k1 = dense ? (uint32_t)((uint64_t)p * n_node + n_node) : cand_off[p + 1];
        int have_best = 0, any_lim = 0; uint32_t fit_k = DRA_GPU_NONE, best_k = 0;
        pair_sum best = { 0 };
        for (uint32_t k = k0; k < k1; k++) {
            uint32_t n = dense ? k - k0 : cand_nodes[k];
            if (n < n_node && cnt <= DRA_MAX_POD)
                for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, n < n_node ? loff[n] : 0,
                               n < n_node ? loff[n + 1] : 0, exh, NULL);
            if (pair_status) pair_status[k] = s.st;
            if (pair_victims) pair_victims[k] = s.st == PRE_EVICT ? s.count : 0;
            if (s.st == PRE_FITS && fit_k == DRA_GPU_NONE) fit_k = k;
            if (s.st == PRE_LIMIT) any_lim = 1;
            if (s.st == PRE_EVICT && (!have_best || better(&s, &best))) { best = s; best_k = k; have_best = 1; }
        }
        uint32_t* row = victims ? victims + (size_t)p * max_victims : NULL;
        for (uint32_t j = 0; j < max_victims; j++) row[j] = DRA_GPU_NONE;
        n_victims[p] = 0;
        if (fit_k != DRA_GPU_NONE) {
            pod_node[p] = dense ? fit_k - k0 : cand_nodes[fit_k];
            pod_status[p] = PRE_FITS;
        } else if (have_best) {
            uint32_t n = dense ? best_k - k0 : cand_nodes[best_k];
            for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, loff[n], loff[n + 1], exh, vic);
            pod_node[p] = n; pod_status[p] = PRE_EVICT; n_victims[p] = s.count;
            for (uint32_t j = 0; j < s.count && j < max_victims; j++) row[j] = vic[j];
        } else {
            int inv = cnt > DRA_MAX_POD;
            for (uint32_t i = 0; i < cnt && !inv; i++) { dra_claim_rec t = claims[c0 + i]; t.node = 0; inv = claim_invalid(&t, 1, 1); }
            pod_node[p] = DRA_GPU_NONE;
            pod_status[p] = inv ? PRE_INVALID : any_lim ? PRE_LIMIT : PRE_NO;
        }
    }
    free(rnode); free(loff); free(list); free(vic);
    return 0;
}
