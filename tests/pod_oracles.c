/*
 * pod_oracles.c — CPU oracles of the pod-level calls: place pods (spec §13), pod capacity (§16), preemption with
 * optional disruption budgets (§14) and preempt and place (§15).  TEST INFRASTRUCTURE ONLY, built by
 * tests/pod_oracles.py.
 *
 * Every evaluation is the §12 pod evaluation of oracle/dra_oracle.c itself (its static pod_eval, included below), and
 * the selectors are its selector state, set once for all four calls.  Restated here: the walk over candidates (§13),
 * the counting loop (§16), the §9 update of a running pod and its inverse, the victim ordering, the budgets' violating
 * flags in the "members of V up to and including v" form, the two-phase reprieve and the choice of the node (§14), and
 * the sequential schedule of §15: pods in input order, each judged on the CURRENT inventory against the running pods
 * not evicted yet, then applied.
 */
#include "../oracle/dra_oracle.c"

#define POD_API __attribute__((visibility("default")))

enum { PRE_FITS = 0, PRE_EVICT = 1, PRE_NO = 2, PRE_LIMIT = 3, PRE_INVALID = 4 };

POD_API void pod_oracle_set_selectors(const dra_gpu_attr* attrs, uint32_t n_gpu, const dra_selector* sels,
                                      uint32_t n_sel)
{
    dra_oracle_set_selectors(attrs, n_gpu, sels, n_sel);
}

/* 1 unless pod_off[0 .. n_pod] starts at 0, ends at n_claim and never decreases */
static int bad_pod_off(const uint32_t* pod_off, uint32_t n_pod, uint32_t n_claim)
{
    if (pod_off[0] != 0 || pod_off[n_pod] != n_claim) return 1;
    for (uint32_t p = 0; p < n_pod; p++) if (pod_off[p + 1] < pod_off[p]) return 1;
    return 0;
}

/* 1: the dense form (cand_nodes == cand_off == NULL, every node ascending); 0: candidate lists, cand_off starting at 0
 * and never decreasing; -1: neither */
static int cand_form(const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t n_pod)
{
    if (cand_nodes == NULL && cand_off == NULL) return 1;
    if (!cand_off || cand_off[0] != 0) return -1;
    for (uint32_t p = 0; p < n_pod; p++) if (cand_off[p + 1] < cand_off[p]) return -1;
    return 0;
}

/* ---- spec §13: place pods ---------------------------------------------------------------------------------------- */

/* Mutates gpus[]; pod_node[p] = the node pod p was placed on, or 0xFFFFFFFF.  cand_nodes == cand_off == NULL: every node,
 * ascending.  flags: DRA_F_EXHAUSTIVE (DRA_F_FRESH_INVENTORY is accepted and has no effect: gpus[] is the starting
 * state).  Returns -1, with nothing changed, on the arguments spec §13 rejects. */
POD_API int pod_oracle_place_pods(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                                  const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                                  const uint32_t* pod_off, uint32_t n_pod,
                                  const uint32_t* cand_nodes, const uint32_t* cand_off,
                                  const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, uint32_t* pod_node,
                                  uint32_t flags)
{
    if (flags & ~(uint32_t)(DRA_F_EXHAUSTIVE | DRA_F_FRESH_INVENTORY)) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (bad_pod_off(pod_off, n_pod, n_claim)) return -1;
    const int dense = cand_form(cand_nodes, cand_off, n_pod);
    if (dense < 0) return -1;
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

/* ---- spec §16: pod capacity -------------------------------------------------------------------------------------- */

/* Evaluations on a private copy of the node that keeps each placement that succeeds.  Returns -1, with nothing written,
 * on the arguments spec §16 rejects.  pair_stop, pod_total and pod_nodes may be NULL. */
POD_API int pod_oracle_capacity(const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                                const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                                const uint32_t* pod_off, uint32_t n_pod,
                                const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t max_copies,
                                uint16_t* pair_copies, uint8_t* pair_stop, uint64_t* pod_total, uint32_t* pod_nodes,
                                uint32_t flags)
{
    if (flags & ~(uint32_t)DRA_F_EXHAUSTIVE) return -1;
    if (max_copies < 1 || max_copies > 65535) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (bad_pod_off(pod_off, n_pod, n_claim)) return -1;
    const int dense = cand_form(cand_nodes, cand_off, n_pod);
    if (dense < 0) return -1;
    if (!dense && cand_off[n_pod] && !cand_nodes) return -1;
    if (dense && (uint64_t)n_pod * n_node >= (1ull << 32)) return -1;
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

/* ---- the running pods and the pair judgement of spec §14 --------------------------------------------------------- */

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

static const int32_t* g_rprio;     /* qsort has no context argument */
static int by_prio_desc(const void* a, const void* b)
{
    uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
    if (g_rprio[x] != g_rprio[y]) return g_rprio[x] > g_rprio[y] ? -1 : 1;
    return x < y ? -1 : x > y;
}

/* Where the running pods are: each one's node is that of its OK slots' GPUs (none without an OK slot).  On success
 * *loff (n_node + 2 entries) and *list (rn_pod + 1) are allocated, node n's running pods being
 * list[loff[n] .. loff[n + 1]) by priority descending, then index.  Returns -1, with nothing allocated, on the running
 * pods spec §14 rejects: a malformed pod_off, a slot range outside rn_out, a GPU index >= n_gpu, OK slots on two
 * nodes. */
static int index_running(const running* R, uint32_t rn_claim, uint32_t rn_pod, uint32_t rn_out, const dra_gpu_rec* gpus,
                         uint32_t n_gpu, uint32_t** loff_out, uint32_t** list_out)
{
    const uint32_t n_node = R->n_node;
    if (bad_pod_off(R->pod_off, rn_pod, rn_claim)) return -1;
    uint32_t* rnode = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    if (!rnode) return -1;
    for (uint32_t r = 0; r < rn_pod; r++) {
        rnode[r] = DRA_GPU_NONE;
        for (uint32_t i = R->pod_off[r]; i < R->pod_off[r + 1]; i++) {
            uint32_t base = R->out_off ? R->out_off[i] : i, sl = run_slots(&R->claims[i], n_node, R->out_off != NULL);
            if (base > rn_out || sl > rn_out - base) { free(rnode); return -1; }
            for (uint32_t k = 0; k < sl; k++) {
                const dra_out_rec* o = &R->out[base + k];
                if (o->status != DRA_ST_OK) continue;
                if (o->gpu >= n_gpu) { free(rnode); return -1; }
                uint32_t n = gpus[o->gpu].node;
                if (rnode[r] == DRA_GPU_NONE) rnode[r] = n;
                else if (rnode[r] != n) { free(rnode); return -1; }
            }
        }
    }
    uint32_t* loff = (uint32_t*)calloc((size_t)n_node + 2, sizeof(uint32_t));
    uint32_t* list = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    if (!loff || !list) { free(rnode); free(loff); free(list); return -1; }
    for (uint32_t r = 0; r < rn_pod; r++) if (rnode[r] < n_node) loff[rnode[r] + 1]++;
    for (uint32_t n = 0; n < n_node; n++) loff[n + 1] += loff[n];
    for (uint32_t r = 0; r < rn_pod; r++) if (rnode[r] < n_node) list[loff[rnode[r]]++] = r;
    for (uint32_t n = n_node; n > 0; n--) loff[n] = loff[n - 1];
    loff[0] = 0;
    g_rprio = R->prio;
    for (uint32_t n = 0; n < n_node; n++) qsort(list + loff[n], loff[n + 1] - loff[n], sizeof(uint32_t), by_prio_desc);
    free(rnode);
    *loff_out = loff; *list_out = list;
    return 0;
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
    uint8_t st; uint32_t count; int32_t hi; uint64_t sum; uint32_t hi_idx; uint32_t viol;
} pair_sum;

/* the budgets: run_pdb[r] (DRA_PDB_NONE: none) and allowed[b]; pdb == NULL: none in force */
typedef struct budgets {
    const uint32_t* pdb; const int32_t* allowed;
} budgets;

/* Pair (pod, node n) under the budgets B: writes the victims (running-pod indices, V order) into vic when non-NULL.  flag:
 * scratch of at least l1 - l0 bytes.  Without budgets no member violates, so the reprieve is one pass in V order and
 * viol is 0. */
static pair_sum judge(const dra_gpu_rec* gpus, const uint32_t* node_off, uint32_t n_node, const dra_profile_tbl* tbl,
                      const dra_claim_rec* pod, uint32_t cnt, int32_t prio, uint32_t n, const running* R,
                      const uint32_t* list, uint32_t l0, uint32_t l1, int exh, uint32_t* vic, const budgets* B,
                      uint8_t* flag)
{
    pair_sum s = { PRE_NO, 0, INT32_MIN, 0, 0xFFFFFFFFu, 0 };
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
    /* flag bit 0: violating (the members of V[v0 .. v] under its budget outnumber what the budget allows); bit 1: victim */
    for (uint32_t v = v0; v < l1; v++) {
        uint32_t b = B->pdb ? B->pdb[list[v]] : DRA_PDB_NONE, members = 0;
        flag[v - l0] = 0;
        if (b == DRA_PDB_NONE) continue;
        for (uint32_t u = v0; u <= v; u++) members += B->pdb[list[u]] == b;
        flag[v - l0] = (int64_t)members > (int64_t)B->allowed[b];
    }
    /* the reprieve: the violating members first, then the others, each in V order */
    for (int phase = 1; phase >= 0; phase--)
        for (uint32_t v = v0; v < l1; v++) {
            if ((flag[v - l0] & 1) != phase) continue;
            memcpy(S2, S, ng * sizeof *S);
            run_apply(R, list[v], S2, g0, ng, 1);
            if (eval_on(S2, g0, ng, tbl, pod, cnt, n_node, exh, &lim)) memcpy(S, S2, ng * sizeof *S);
            else flag[v - l0] |= 2;
        }
    for (uint32_t v = v0; v < l1; v++) {                 /* the victims, in V order */
        uint32_t r = list[v];
        if (!(flag[v - l0] & 2)) continue;
        if (s.count == 0 || R->prio[r] > s.hi) { s.hi = R->prio[r]; s.hi_idx = r; }   /* V order: the lowest index first */
        s.sum += (uint64_t)((int64_t)R->prio[r] + 2147483648ll);
        s.viol += flag[v - l0] & 1;
        if (vic) vic[s.count] = r;
        s.count++;
    }
    return s;
}

/* 1 when a is preferred to b (pickOneNodeForPreemption without start times) */
static int better(const pair_sum* a, const pair_sum* b)
{
    if (a->viol != b->viol) return a->viol < b->viol;
    if (a->hi != b->hi) return a->hi < b->hi;
    if (a->sum != b->sum) return a->sum < b->sum;
    if (a->count != b->count) return a->count < b->count;
    if (a->hi_idx != b->hi_idx) return a->hi_idx > b->hi_idx;
    return 0;                                            /* equal: the earlier candidate stays */
}

/* ---- spec §14: preemption, with disruption budgets --------------------------------------------------------------- */

/* Every pair judged on a private copy of the node.  Returns -1, with nothing written, on the arguments spec §14
 * rejects.  run_pdb / allowed / n_pdb: the budgets (NULL and 0: none); pair_viol and pod_viol may be NULL. */
POD_API int pod_oracle_preempt(const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
                               const dra_profile_tbl* tbl, const dra_claim_rec* claims, uint32_t n_claim,
                               const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                               const uint32_t* cand_nodes, const uint32_t* cand_off,
                               const dra_claim_rec* rclaims, uint32_t rn_claim, const uint32_t* rpod_off,
                               const int32_t* rprio, uint32_t rn_pod, const uint32_t* rout_off,
                               const dra_out_rec* rout, uint32_t rn_out,
                               const uint32_t* run_pdb, const int32_t* allowed, uint32_t n_pdb,
                               uint8_t* pair_status, uint32_t* pair_victims, uint32_t* pair_viol,
                               uint32_t* pod_node, uint8_t* pod_status, uint32_t* n_victims, uint32_t* pod_viol,
                               uint32_t* victims, uint32_t max_victims, uint32_t flags)
{
    if (flags & ~(uint32_t)DRA_F_EXHAUSTIVE) return -1;
    if (n_pdb && !allowed) return -1;
    if (check_inventory(gpus, n_gpu, node_off, n_node, tbl)) return -1;
    if (bad_pod_off(pod_off, n_pod, n_claim)) return -1;
    const int dense = cand_form(cand_nodes, cand_off, n_pod);
    if (dense < 0) return -1;
    if (dense && (uint64_t)n_pod * n_node >= (1ull << 32)) return -1;
    if (max_victims && !victims) return -1;
    if (n_pod == 0) return 0;                            /* no pending pods: the running pods are not examined */
    if (n_pdb && rn_pod && !run_pdb) return -1;
    for (uint32_t r = 0; run_pdb && r < rn_pod; r++) if (run_pdb[r] != DRA_PDB_NONE && run_pdb[r] >= n_pdb) return -1;
    const budgets B = { n_pdb ? run_pdb : NULL, allowed };
    const running R = { rclaims, rpod_off, rprio, rout_off, rout, n_node };
    uint32_t *loff, *list;
    if (index_running(&R, rn_claim, rn_pod, rn_out, gpus, n_gpu, &loff, &list)) return -1;
    uint32_t* vic = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    uint8_t* flag = (uint8_t*)malloc((size_t)rn_pod + 1);
    if (!vic || !flag) { free(loff); free(list); free(vic); free(flag); return -1; }

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
                               n < n_node ? loff[n + 1] : 0, exh, NULL, &B, flag);
            if (pair_status) pair_status[k] = s.st;
            if (pair_victims) pair_victims[k] = s.st == PRE_EVICT ? s.count : 0;
            if (pair_viol) pair_viol[k] = s.st == PRE_EVICT ? s.viol : 0;
            if (s.st == PRE_FITS && fit_k == DRA_GPU_NONE) fit_k = k;
            if (s.st == PRE_LIMIT) any_lim = 1;
            if (s.st == PRE_EVICT && (!have_best || better(&s, &best))) { best = s; best_k = k; have_best = 1; }
        }
        uint32_t* row = victims ? victims + (size_t)p * max_victims : NULL;
        for (uint32_t j = 0; j < max_victims; j++) row[j] = DRA_GPU_NONE;
        n_victims[p] = 0;
        if (pod_viol) pod_viol[p] = 0;
        if (fit_k != DRA_GPU_NONE) {
            pod_node[p] = dense ? fit_k - k0 : cand_nodes[fit_k];
            pod_status[p] = PRE_FITS;
        } else if (have_best) {
            uint32_t n = dense ? best_k - k0 : cand_nodes[best_k];
            for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, loff[n], loff[n + 1], exh, vic,
                               &B, flag);
            pod_node[p] = n; pod_status[p] = PRE_EVICT; n_victims[p] = s.count;
            if (pod_viol) pod_viol[p] = s.viol;
            for (uint32_t j = 0; j < s.count && j < max_victims; j++) row[j] = vic[j];
        } else {
            int inv = cnt > DRA_MAX_POD;
            for (uint32_t i = 0; i < cnt && !inv; i++) { dra_claim_rec t = claims[c0 + i]; t.node = 0; inv = claim_invalid(&t, 1, 1); }
            pod_node[p] = DRA_GPU_NONE;
            pod_status[p] = inv ? PRE_INVALID : any_lim ? PRE_LIMIT : PRE_NO;
        }
    }
    free(loff); free(list); free(vic); free(flag);
    return 0;
}

/* ---- spec §15: preempt and place --------------------------------------------------------------------------------- */

/* Mutates gpus[].  cand_nodes == cand_off == NULL: every node, ascending.  No budgets.  Returns -1, with nothing
 * written and gpus[] unchanged, on the arguments spec §15 rejects. */
POD_API int pod_oracle_preempt_place(dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node,
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
    if (bad_pod_off(pod_off, n_pod, n_claim)) return -1;
    const int dense = cand_form(cand_nodes, cand_off, n_pod);
    if (dense < 0) return -1;
    for (uint32_t p = 0; !dense && p < n_pod; p++) if (cand_off[p + 1] - cand_off[p] > POS_MAX) return -1;
    if (dense && (uint64_t)n_pod * n_node >= (1ull << 32)) return -1;
    const int have_off = out_off != NULL;
    for (uint32_t i = 0; i < n_claim; i++) {              /* slots as if the claim named a node of the inventory */
        dra_claim_rec t = claims[i]; t.node = 0;
        uint32_t b = have_off ? out_off[i] : i, sl = claim_slots(&t, 1, have_off);
        if (b > n_out || sl > n_out - b) return -1;
    }
    if (n_pod == 0) return 0;                             /* no pending pods: the running pods are not examined */
    const budgets none = { NULL, NULL };
    const running R = { rclaims, rpod_off, rprio, rout_off, rout, n_node };
    /* per node: its running pods not evicted yet, by priority descending, then index: list[loff[n] .. lend[n]) */
    uint32_t *loff, *list;
    if (index_running(&R, rn_claim, rn_pod, rn_out, gpus, n_gpu, &loff, &list)) return -1;
    uint32_t* lend = (uint32_t*)malloc(((size_t)n_node + 1) * sizeof(uint32_t));
    uint32_t* vic = (uint32_t*)malloc(((size_t)rn_pod + 1) * sizeof(uint32_t));
    uint8_t* flag = (uint8_t*)malloc((size_t)rn_pod + 1);
    if (!lend || !vic || !flag) { free(loff); free(list); free(lend); free(vic); free(flag); return -1; }
    for (uint32_t n = 0; n < n_node; n++) lend[n] = loff[n + 1];
    for (uint32_t r = 0; r < rn_pod; r++) evicted_by[r] = DRA_GPU_NONE;

    const int exh = (flags & DRA_F_EXHAUSTIVE) != 0;
    dra_claim_rec pod[DRA_MAX_POD];
    for (uint32_t p = 0; p < n_pod; p++) {
        uint32_t c0 = pod_off[p], cnt = pod_off[p + 1] - c0;
        uint32_t k0 = dense ? 0 : cand_off[p], k1 = dense ? n_node : cand_off[p + 1];
        int have_best = 0, any_lim = 0; uint32_t fit_k = DRA_GPU_NONE, best_k = 0;
        pair_sum best = { 0 };
        /* a claim invalid in the call's slot mode: INVALID, judged nowhere (judge() assumes out_off) */
        int inv = cnt > DRA_MAX_POD;
        for (uint32_t i = 0; i < cnt && !inv; i++) { dra_claim_rec t = claims[c0 + i]; t.node = 0; inv = claim_invalid(&t, 1, have_off); }
        if (inv) k1 = k0;
        for (uint32_t k = k0; k < k1; k++) {              /* §14's pairs on the current state */
            uint32_t n = dense ? k : cand_nodes[k];
            if (n < n_node && cnt <= DRA_MAX_POD)
                for (uint32_t i = 0; i < cnt; i++) { pod[i] = claims[c0 + i]; pod[i].node = n; }
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, n < n_node ? loff[n] : 0,
                               n < n_node ? lend[n] : 0, exh, NULL, &none, flag);
            if (s.st == PRE_FITS && fit_k == DRA_GPU_NONE) fit_k = k;
            if (s.st == PRE_LIMIT) any_lim = 1;
            if (s.st == PRE_EVICT && (!have_best || better(&s, &best))) { best = s; best_k = k; have_best = 1; }
        }
        uint32_t n = DRA_GPU_NONE;
        if (fit_k != DRA_GPU_NONE) { n = dense ? fit_k : cand_nodes[fit_k]; pod_status[p] = PRE_FITS; }
        else if (have_best) { n = dense ? best_k : cand_nodes[best_k]; pod_status[p] = PRE_EVICT; }
        else pod_status[p] = inv ? PRE_INVALID : any_lim ? PRE_LIMIT : PRE_NO;
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
            pair_sum s = judge(gpus, node_off, n_node, tbl, pod, cnt, prio[p], n, &R, list, loff[n], lend[n], exh, vic,
                               &none, flag);
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
    free(loff); free(list); free(lend); free(vic); free(flag);
    return 0;
}
