// dra_api.cu — C ABI of libdra_alloc.so (include/dra_alloc.h): context, staging, kernel chain, NCCL.
//
// No CPU fallback lives here: every entry point that computes anything launches the sm_90a kernels of
// dra_device.cuh, and dra_ctx_create fails when there is no usable device.
#include "dra_device.cuh"

#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <vector>

using namespace dra;

namespace {

thread_local std::string g_create_err;

// registry of dra_host_alloc buffers: passing one of these skips the staging copy
std::mutex g_pin_mu;
std::map<uintptr_t, size_t> g_pinned;

bool is_pinned(const void* p, size_t bytes) {
    if (!p) return false;
    std::lock_guard<std::mutex> lk(g_pin_mu);
    auto it = g_pinned.upper_bound((uintptr_t)p);
    if (it == g_pinned.begin()) return false;
    --it;
    return (uintptr_t)p + bytes <= it->first + it->second;
}

struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool load(std::string& err) {
        if (lib) return true;
        // libnccl.so.2 already mapped by the host runtime (torch) is reused by soname
        lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) { err = std::string("dlopen libnccl: ") + dlerror(); return false; }
        GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
        AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
        CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
        GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
        if (!GetUniqueId || !CommInitRank || !AllGather || !CommDestroy) { err = "libnccl: missing symbols"; return false; }
        return true;
    }
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

}  // namespace

// A peer exchange's region of the peer buffer (dra_device.cuh PeerExchange): [staging x2 by call parity][flag words].
// slice: the bytes of one sender's slice of the staging (0: every sender writes at global indices, as the sync does).
struct PeerRegion {
    size_t stage[2] = {0, 0}, flags = 0, slice = 0;
    uint32_t seq = 0;             // the exchange's last call
};

// The sizes the sharded calls' peer exchanges are reserved for, one group per dra_set_shard_* setter
struct ShardSizes {
    uint32_t uns_pairs;                             // dra_set_shard_pairs
    uint32_t place_pods;                            // dra_set_shard_place
    uint32_t pre_pods, pre_pairs, pre_victims;      // dra_set_shard_preempt
    uint32_t scap_pairs;                            // dra_set_shard_capacity
    uint32_t spp_pods, spp_pairs, spp_run;          // dra_set_shard_preempt_place
    uint32_t swhy_pairs;                            // dra_set_shard_why
};

struct dra_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    uint32_t cfg_flags = 0;

    // inventory
    uint32_t n_gpu = 0, n_node = 0, max_width = 0;     // max_width: most GPUs on one node
    uint4* d_inv_live = nullptr;
    uint4* d_inv_pristine = nullptr;
    uint32_t* d_node_off = nullptr;
    uint32_t* d_tbl = nullptr;
    dra_profile_tbl h_tbl[DRA_MAX_MODELS];
    bool tbl_dirty = true;
    uint4* d_attrs = nullptr;  uint32_t n_attr = 0;      // spec §10
    uint4* d_sels = nullptr;   uint32_t n_sel = 0;

    // batch buffers (device)
    size_t cap_claims = 0, cap_out = 0, cap_hist = 0, cap_nodes = 0, cap_pairs = 0, cap_pods = 0, cap_bits_only = 0;
    uint4* d_claims = nullptr;
    uint4* d_sorted = nullptr;
    uint32_t* d_out_off = nullptr;
    uint2* d_out = nullptr;
    uint16_t* d_rank = nullptr;
    uint32_t* d_hist = nullptr;
    uint32_t* d_claim_off = nullptr;
    uint32_t *d_pod_off = nullptr, *d_cand_off = nullptr, *d_cand_nodes = nullptr, *d_pair_pod = nullptr, *d_bits = nullptr;
    uint4* d_podrec = nullptr; size_t cap_podrec = 0;     // pod mode (spec §12); place pods (§13): the pair records
    uint32_t *d_place_state = nullptr, *d_place_node = nullptr; size_t cap_place_pods = 0;   // place pods: per pod
    uint32_t* d_place_cursor = nullptr; size_t cap_place_cursor = 0;                          // place pods: per node (+ 1)
    int place_occ = -1;                   // resident CTAs of k_pods_place<4> per SM (occupancy query, once)
    int place_why_occ = -1;               // resident CTAs of k_pods_place<4, false, true> per SM (dra_place_pods_why_batch)
    // preemption (spec §14): per pending pod, per pair, the running pods and the victim rows
    uint32_t *d_pre_prio = nullptr, *d_pre_node = nullptr, *d_pre_nvic = nullptr, *d_pre_choice = nullptr; uint8_t* d_pre_pst = nullptr;
    uint32_t* d_pre_podviol = nullptr; size_t cap_pre_pods = 0;
    uint4* d_pre_psum = nullptr; unsigned long long* d_pre_psum64 = nullptr; uint8_t* d_pre_pairst = nullptr;
    uint32_t *d_pre_pairvic = nullptr, *d_pre_pairviol = nullptr; size_t cap_pre_pairs = 0;
    uint4* d_pre_rclaims = nullptr; uint32_t* d_pre_routoff = nullptr; size_t cap_pre_rclaims = 0;
    uint32_t *d_pre_rpodoff = nullptr, *d_pre_rprio = nullptr; uint4 *d_pre_rrec = nullptr, *d_pre_vlist = nullptr;
    uint32_t *d_pre_rpdb = nullptr, *d_pre_vprev = nullptr; size_t cap_pre_rpods = 0;   // budgets: run_pdb, vprev
    int32_t* d_pre_allowed = nullptr; size_t cap_pre_allowed = 0;                        // budgets: disruptionsAllowed
    uint2* d_pre_rout = nullptr; size_t cap_pre_rout = 0;
    uint32_t* d_pre_vic = nullptr; size_t cap_pre_vic = 0;
    // preempt and place (spec §15): per pending pod, per running pod, per node (the running lists' offsets, the last pod
    // judged there)
    uint32_t* d_pp_pending = nullptr; size_t cap_pp_pods = 0;
    uint32_t* d_pp_evicted = nullptr; size_t cap_pp_rpods = 0;
    uint32_t *d_pp_runoff = nullptr, *d_pp_judged = nullptr; size_t cap_pp_nodes = 0;
    int pp_occ = -1;                      // resident CTAs of k_pods_preempt_place<4> per SM (occupancy query, once)
    int pp_why_occ = -1;                  // resident CTAs of k_pods_preempt_place<4, true> per SM (dra_preempt_place_why_batch)
    // pod capacity (spec §16): per pair, per pod
    uint16_t* d_cap_copies = nullptr; uint8_t* d_cap_stop = nullptr; size_t cap_cap_pairs = 0;
    unsigned long long* d_cap_total = nullptr; uint32_t* d_cap_nodes = nullptr; size_t cap_cap_pods = 0;
    uint8_t* d_why = nullptr; uint32_t* d_why_claim = nullptr; size_t cap_why_pairs = 0;      // dra_unsuitable_why_batch
    uint32_t* d_why_pod = nullptr; size_t cap_why_pods = 0; uint32_t* d_why_blocks = nullptr; size_t cap_why_claims = 0;

    // error flags
    uint32_t* d_err = nullptr;            // device memory
    volatile uint32_t* h_err = nullptr;   // mapped pinned host memory
    uint32_t* h_err_dev = nullptr;        // device alias of h_err

    // pinned staging
    uint8_t* h_in = nullptr;  size_t h_in_cap = 0;
    uint8_t* h_out = nullptr; size_t h_out_cap = 0;

    uint64_t launches = 0;
    uint32_t chain = 0, chain_tile = 0;   // DRA_K_* bits and hist tile of the last Allocate-family call (dra_debug_last_chain)
    bool profiling = false;
    cudaEvent_t ev[8] = {};
    bool ev_ok = false;
    float timings[5] = {0, 0, 0, 0, 0};
    uint32_t ev_mask = 0;
    uint64_t fused_max_work = 3000000ull;   // n_node * n_claim up to which the single-launch kernel is used
    uint32_t fused_max_one_wave = 14000u, fused_max_multi = 7500u;   // claims up to which it beats the sort path (profiles/path_crossover.py,
                                                                     // fused_plan); dra_calibrate re-measures them on the device at hand
    // direct host I/O of the single-launch kernel (DirectIO in dra_device.cuh)
    DirectIO dio_pending{};                 // set by dra_allocate_batch for the next launch_allocate, then cleared
    uint32_t* d_gbar = nullptr;             // grid barrier words
    int n_sm = 0, coop_ok = 0;
    int fused_occ_stage = -1, fused_occ_smem = -1, fused_occ_cta = 0;   // fused_resident_ctas: the last query's answer
    unsigned long long* d_scan_status = nullptr; uint32_t cap_scan_status = 0;   // k_bucket_scan_rows: one word per CTA
    int pack4_occ = -1;              // resident CTAs of k_pack<4> per SM (occupancy query, once)
    const void* dio_seen[3] = {nullptr, nullptr, nullptr};   // host pointers already checked to be device-visible as-is

    ncclComm_t comm = nullptr;
    int rank = 0, world = 1;

    // resident mode (k_serve): the single-launch kernel stays up and takes batches by doorbell
    bool serve_on = false;
    cudaStream_t serve_stream = nullptr;
    ServeCmd* h_cmd = nullptr; ServeCmd* h_cmd_dev = nullptr;          // mapped host memory (one cache line)
    volatile uint32_t* h_stat = nullptr; uint32_t* h_stat_dev = nullptr;
    uint32_t* d_go = nullptr;
    uint32_t serve_seq = 0, serve_cap = 0; size_t serve_smem = 0; uint64_t serve_epoch = 0;
    uint64_t serve_batches = 0;

    // CUDA-graph replay of the host-buffer Allocate call
    struct GraphKeyT { const void* c; const void* o; void* d; uint32_t n_claim, n_out, flags; uint64_t epoch;
                       bool operator==(const GraphKeyT& k) const { return c == k.c && o == k.o && d == k.d && n_claim == k.n_claim && n_out == k.n_out && flags == k.flags && epoch == k.epoch && c != nullptr; } };
    GraphKeyT graph_key{};
    cudaGraphExec_t graph_exec = nullptr;
    uint32_t graph_launches = 0, graph_chain = 0, graph_tile = 0;
    uint64_t state_epoch = 1;     // bumped by every call that reallocates or re-points device state

    // peer-memory all-gather (packets over NVLink, dra_device.cuh PktGather)
    bool peer_ready = false;
    uint32_t peer_form = 0;                     // 1: per-rank slices [world][n_per]   2: global slots [tab_len]
    uint32_t peer_n_per = 0, peer_tab_len = 0, peer_cap = 0, peer_epoch = 0;
    size_t peer_bytes = 0, off_table[2] = {0, 0}, off_stage[2] = {0, 0}, off_hdr[2] = {0, 0};
    PeerRegion rendezvous_x, uns_x, isync_x;    // the peer exchanges: rendezvous (flags alone), UnsuitableNodes, inventory sync
    uint8_t* peer_local = nullptr;              // this rank's buffer (cudaMalloc, exported by IPC handle)
    uint8_t* peer_base[PEER_MAX] = {};          // every rank's buffer as mapped here
    bool peer_ipc[PEER_MAX] = {};               // mapped with cudaIpcOpenMemHandle (else: same process)
    uint32_t* d_cursor = nullptr;               // [2] packet reservation cursors (local)
    long long peer_spin = 4000000000ll;         // cycles a receiver waits for a packet before ERR_PEER_TIMEOUT
    // sharded global batch
    bool shard_on = false; uint32_t shard_lo = 0, shard_hi = 0, shard_stray = 0, shard_epoch = 0;
    unsigned long long* d_sc_times = nullptr;   // instrumentation (DRA_TIMELINE)
    uint32_t shard_last_n = 0;                  // batch size of the last sharded call (the plan hint is per batch size)
    bool shard_map_on = false; uint32_t shard_bounds[PEER_MAX + 1] = {}; uint32_t shard_stray_rank = 0;
    uint32_t* d_rank_slots = nullptr;           // [2][PEER_MAX] OutRec slots per rank, counted by the compaction
    uint4* d_cclaims = nullptr; uint32_t* d_coff = nullptr; size_t cap_cclaims = 0;
    unsigned long long* d_sc_status = nullptr; size_t cap_sc_status = 0;
    uint32_t* d_sc_counts = nullptr;            // device: [0] claims kept, [1] slots
    volatile uint32_t* h_sc_counts = nullptr;   // mapped host copy of the last call's counts
    uint32_t* h_sc_counts_dev = nullptr;
    uint2* d_gtable = nullptr; size_t cap_gtable = 0;   // result table when no peers are set up (world 1)
    uint32_t* d_ticket = nullptr;               // 16 words, zeroed when allocated (dra_ctx_create): see Ticket
    ShardSizes shard_req{};                     // the sizes the setters asked for, reserved by the next peer_setup
    ShardSizes shard_rsv{};                     // the sizes the last peer_setup reserved
    // sharded UnsuitableNodes: bit exchange in the peer buffer ([staging x2: world slices of uns_stride words][flags])
    uint32_t uns_stride = 0;
    uint32_t* d_ubits = nullptr; size_t cap_ubits = 0;   // this rank's words of the call
    uint32_t* d_upair_pod = nullptr; size_t cap_upair_pod = 0;   // candidate form: pair -> pod (k_uns_prep)
    // sharded pods Allocate
    uint32_t* d_spod = nullptr;                 // [SP_WORDS] call words (dra_device.cuh SPodArgs)
    // sharded place pods: a region [progress counter, 64 bytes][state words: u64 per pod] (dra_device.cuh PlaceShard) in
    // the peer buffer at world > 1, in d_splace_local at world 1
    size_t off_splace = 0;
    uint8_t* d_splace_local = nullptr; size_t cap_splace_local = 0;    // pods
    uint32_t splace_seq = 0;                    // the last call's sequence number (peer_setup starts over: fresh words)
    uint4* d_splace_rec = nullptr; size_t cap_splace_rec = 0;          // [n_pod] finaliser records for k_spod_gather
    // sharded preemption: a region [partials x2: world slices][flags] (dra_device.cuh PreShard) in the peer buffer
    PeerRegion pre_x;
    uint4* d_spre_part = nullptr; size_t cap_spre_part = 0;           // this rank's partials and pair results (uint4 units)
    // sharded preempt and place: the world's state assembled for the call (scratch inventory), and the call's gate word
    uint4* d_spp_inv = nullptr; size_t cap_spp_inv = 0;
    uint32_t* d_spp_gate = nullptr;
    PeerRegion spp_x;                           // the verdict agreement's flags (k_spp_agree), after the exchange
    // sharded pod capacity: a region [slices x2: world slices][flags] (dra_device.cuh CapMerge) in the peer buffer
    PeerRegion scap_x;
    uint4* d_scap_part = nullptr; size_t cap_scap_part = 0;           // this rank's slice (uint4 units)
    // sharded reasons of UnsuitableNodes: a region [slices x2: world slices][flags] (dra_device.cuh WhyMerge) in the peer buffer
    PeerRegion swhy_x;
    uint4* d_swhy_part = nullptr; size_t cap_swhy_part = 0;           // this rank's slice (uint4 units)
    uint32_t* d_swhy_blocks = nullptr; size_t cap_swhy_blocks = 0;    // the merge's per-claim counts and blocks-done counter
    int splace_occ = -1;                        // resident CTAs of k_pods_place<4, true> per SM (occupancy query, once)
    int splace_why_occ = -1;                    // resident CTAs of k_pods_place<4, true, true> per SM (sharded §18)
    int peers_on_device = 1;                    // ranks whose contexts share this device (dra_peer_import_local)
    // inventory sync: records in the peer buffer ([staging x2: peer_inv_gpus records][flags[PEER_MAX], elect[2]])
    uint32_t peer_inv_gpus = 0;                 // n_gpu when the export ran (0: no inventory then)
    std::vector<uint32_t> h_node_off;           // host copy of the inventory's node_off: each rank's GPU range
    // Buffers a sharded call outgrew while peers on this device may be waiting for it: cudaFree would wait for the whole
    // device, so they are freed at the next dra_ctx_sync instead (grow / grow_nc while defer_free is set).
    bool defer_free = false;
    std::vector<void*> retired;
    unsigned long long* d_timeline = nullptr; size_t tl_cap = 0; uint32_t tl_n = 0;
    const dra_out_rec* gather_table = nullptr;  // where the last gather's complete table lives (device)
    uint32_t gather_n_per = 0, gather_len = 0;   // gather_len != 0: a global table of that many records

    std::string err;
};

using GraphKey = dra_ctx::GraphKeyT;

namespace {

int fail(dra_ctx* c, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    if (c) c->err = buf; else g_create_err = buf;
    return code;
}

#define CU(call)                                                                                       \
    do { cudaError_t e_ = (call);                                                                     \
         if (e_ != cudaSuccess) return fail(ctx, DRA_E_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)

// The words of d_ticket: the shard compaction's tile ticket, k_bucket_scan8's ticket, k_bucket_scan_rows' ticket and epoch
// (two words), and the 64-bit counters of the counter walks (walk_counter, two words each)
enum Ticket : int { TK_COMPACT = 4, TK_WALK_PREEMPT = 6, TK_SCAN8 = 8, TK_SCAN_ROWS = 10, TK_WALK_UNSUITABLE = 12, TK_WALK_CAPACITY = 14 };

// The 64-bit walk counter at d_ticket word `word` (even: 8-aligned), zeroed on the stream for the walk about to be
// enqueued.  64 bits because a walk may cover up to 2^32 - 1 pairs and every warp takes one more value past its end: a
// 32-bit counter would wrap and walk the pairs again.
int walk_counter(dra_ctx* ctx, Ticket word, unsigned long long*& work) {
    work = reinterpret_cast<unsigned long long*>(ctx->d_ticket + word);
    CU(cudaMemsetAsync(work, 0, 8, ctx->stream));
    return DRA_OK;
}

template <class T>
int grow(dra_ctx* ctx, T*& p, size_t& cap, size_t need, size_t slack = 16) {
    if (need <= cap && p) return DRA_OK;
    size_t ncap = std::max(need, cap + cap / 2) + slack;
    if (p && ctx->defer_free) ctx->retired.push_back(p);
    else if (p) CU(cudaFree(p));
    p = nullptr;
    CU(cudaMalloc((void**)&p, ncap * sizeof(T)));
    cap = ncap;
    ctx->state_epoch++;
    return DRA_OK;
}

template <class T>
int grow_nc(dra_ctx* ctx, T*& p, size_t have_cap, size_t new_cap) {   // companion buffer, cap tracked elsewhere
    if (p && new_cap <= have_cap) return DRA_OK;
    if (p && ctx->defer_free) ctx->retired.push_back(p);
    else if (p) CU(cudaFree(p));
    p = nullptr;
    CU(cudaMalloc((void**)&p, new_cap * sizeof(T)));
    ctx->state_epoch++;
    return DRA_OK;
}

// A group of buffers that share the capacity cap (elements): once need exceeds it, every one of them is reallocated for
// need + need / 2 + 64 elements.  A sharded call and its dra_shard_export compute need through the same function, so the
// export leaves nothing for the call to outgrow.
template <class... T>
int grow_set(dra_ctx* ctx, size_t& cap, size_t need, T*&... bufs) {
    if (need <= cap) return DRA_OK;
    const size_t ncap = need + need / 2 + 64;
    int rc = DRA_OK;
    ((rc = rc ? rc : grow_nc(ctx, bufs, 0, ncap)), ...);
    if (rc) return rc;
    cap = ncap;
    return DRA_OK;
}

int grow_pinned(dra_ctx* ctx, uint8_t*& p, size_t& cap, size_t need) {
    if (need <= cap && p) return DRA_OK;
    size_t ncap = std::max(need, cap + cap / 2) + 256;
    if (p) CU(cudaFreeHost(p));
    p = nullptr;
    CU(cudaHostAlloc((void**)&p, ncap, cudaHostAllocDefault));
    cap = ncap;
    return DRA_OK;
}

struct Tiling { uint32_t T, n_tiles; bool cta_wide; };
Tiling tiling(uint32_t n_claim, uint32_t n_node, int n_sm) {
    // CTA-wide tiles (k_bucket_hist8) whenever 8 x (n_node+1) u16 counters fit in shared memory: 2048 claims, or — once
    // such tiles would outnumber the SMs — the multiple of 2048 that fills the SMs once (<= 32768: ranks are u16)
    if ((size_t)8 * ((size_t)n_node + 2) * 2 <= 200 * 1024) {
        uint32_t T = H8_TILE;
        if (n_claim > (uint32_t)n_sm * H8_TILE)
            T = std::min<uint32_t>(32768u, ((n_claim + (uint32_t)n_sm - 1) / (uint32_t)n_sm + H8_TILE - 1) / H8_TILE * H8_TILE);
        uint32_t n_tiles = n_claim ? (n_claim + T - 1) / T : 1;
        return {T, n_tiles, true};
    }
    uint32_t T = (n_claim + 63) / 64;
    T = (T + 31) & ~31u;
    T = std::max(256u, std::min(T, 65504u));
    uint32_t n_tiles = n_claim ? (n_claim + T - 1) / T : 1;
    return {T, n_tiles, false};
}

int ensure_batch(dra_ctx* ctx, uint32_t n_claim, uint32_t n_out, bool own_io) {
    size_t need_c = std::max<size_t>(n_claim, 1), need_o = std::max<size_t>(n_out, 1);
    if (need_c > ctx->cap_claims || !ctx->d_sorted) {
        size_t ncap = std::max(need_c, ctx->cap_claims + ctx->cap_claims / 2) + 64;
        int rc;
        if ((rc = grow_nc(ctx, ctx->d_claims, 0, ncap))) return rc;
        if ((rc = grow_nc(ctx, ctx->d_sorted, 0, ncap))) return rc;
        if ((rc = grow_nc(ctx, ctx->d_out_off, 0, ncap))) return rc;
        if ((rc = grow_nc(ctx, ctx->d_rank, 0, ncap))) return rc;
        ctx->cap_claims = ncap;
    }
    if (own_io) { int rc = grow(ctx, ctx->d_out, ctx->cap_out, need_o, 64); if (rc) return rc; }
    // d_hist for a sort of any record count up to n_claim (the pod calls sort fewer records than they stage claims).  The
    // tile count is not monotone in the count: tiles grow once there would be more than n_sm CTA-wide tiles (or 64
    // one-warp tiles), so n_sm * 2048 records take n_sm tiles where more records can take fewer.
    Tiling t = tiling(n_claim, ctx->n_node, ctx->n_sm);
    const size_t knee = t.cta_wide ? std::min<size_t>(ctx->n_sm, ((size_t)n_claim + H8_TILE - 1) / H8_TILE)
                                   : std::min<size_t>(64, ((size_t)n_claim + 255) / 256);
    size_t need_h = std::max<size_t>(t.n_tiles, knee) * (ctx->n_node + 1);
    int rc = grow(ctx, ctx->d_hist, ctx->cap_hist, need_h, 64);
    if (rc) return rc;
    // k_bucket_scan_rows: one status word per CTA of 32 nodes, zeroed once (here, never inside a stream capture)
    const uint32_t n_cta = (ctx->n_node + 1 + 31) / 32;
    if (ctx->cap_scan_status < n_cta) {
        CU(cudaStreamSynchronize(ctx->stream));
        if (ctx->d_scan_status && ctx->defer_free) ctx->retired.push_back(ctx->d_scan_status);
        else if (ctx->d_scan_status) CU(cudaFree(ctx->d_scan_status));
        ctx->d_scan_status = nullptr; ctx->cap_scan_status = 0;
        const uint32_t ncap = n_cta + n_cta / 2 + 64;
        CU(cudaMalloc((void**)&ctx->d_scan_status, (size_t)ncap * 8));
        CU(cudaMemset(ctx->d_scan_status, 0, (size_t)ncap * 8));
        ctx->cap_scan_status = ncap;
        ctx->state_epoch++;
    }
    return DRA_OK;
}

SelCtx sel_of(dra_ctx* ctx) { return SelCtx{ctx->n_attr == ctx->n_gpu ? ctx->d_attrs : nullptr, ctx->d_sels, ctx->n_sel}; }

Err err_of(dra_ctx* ctx) { return Err{ctx->d_err, (volatile uint32_t*)ctx->h_err_dev}; }

int upload_table(dra_ctx* ctx) {
    if (!ctx->tbl_dirty) return DRA_OK;
    CU(cudaMemcpyAsync(ctx->d_tbl, ctx->h_tbl, sizeof ctx->h_tbl, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));   // h_tbl is pageable; keep it simple (rare call)
    ctx->tbl_dirty = false;
    return DRA_OK;
}

// Kernel launch with at most one launch attribute.  LA_PDL (programmatic dependent launch): the kernel's CTAs may be
// scheduled while its predecessor in the stream drains; it blocks in griddepcontrol.wait until that grid has completed.
// LA_COOP (cooperative launch): every CTA of the grid is resident at once, or the launch fails.
enum LaunchAttr { LA_NONE, LA_PDL, LA_COOP };
template <typename... KA, typename... A>
static cudaError_t launch_k(void (*k)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, LaunchAttr la, A&&... args) {
    cudaLaunchConfig_t lc; memset(&lc, 0, sizeof lc);
    lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = smem; lc.stream = st;
    cudaLaunchAttribute at[1];
    if (la == LA_PDL) { at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1; }
    else { at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1; }
    lc.attrs = at; lc.numAttrs = la == LA_NONE ? 0u : 1u;
    return cudaLaunchKernelEx(&lc, k, static_cast<KA>(args)...);
}

// A kernel that follows another in the stream is its programmatic dependent (its launch latency and prologue overlap the
// predecessor's tail), except while per-kernel events are being recorded
LaunchAttr pdl_attr(const dra_ctx* ctx) { return ctx->profiling ? LA_NONE : LA_PDL; }

struct Prof {          // event i brackets stage i: [hist, scan, scatter, pack/fused, all-gather]
    dra_ctx* c; int i = 0;
    explicit Prof(dra_ctx* ctx) : c(ctx) { c->ev_mask = 0; rec(0); }
    void rec(int k) { if (c->profiling) { cudaEventRecord(c->ev[k], c->stream); c->ev_mask |= 1u << k; } i = k; }
    void mark() { rec(i + 1); }
    void skip_to(int k) { rec(k); }      // stages before k did not run in this call
};

// The kernel chain of one Allocate batch on device-resident inputs.  Enqueues only.
constexpr int FUSED_NW = 8;
// Which kernel chain an Allocate batch takes.  Small batches: ONE launch — every node's CTA filters the claim
// stream for itself (n_node * n_claim key tests spread over n_node SMs, data from L2) and packs; no sort, no copy.
struct FusedPlan { bool fused, stage; size_t smem; };
FusedPlan fused_plan(const dra_ctx* ctx, uint32_t n_claim, uint32_t flags, uint32_t n_node) {
    FusedPlan p;
    p.stage = n_claim <= FUSED_NW * FU_PIECE * FU_MAXPIECE && fused_smem_bytes(n_claim, FUSED_NW, true) <= 225 * 1024;
    p.smem = fused_smem_bytes(n_claim, FUSED_NW, p.stage);
    // Measured crossover against the sort path (profiles/path_crossover.py, H100 SXM at 700 W): with 125 nodes (one wave
    // of CTAs) the single launch takes 15-19 us up to 12,000 claims against 21-23 us for the sort path; with 250 nodes
    // (two waves) 19.7 against 22.2 us at 6,000 claims.  The single launch grows faster with the claim count.
    const uint32_t fused_max_claims = (int)(n_node + 1) <= ctx->n_sm ? ctx->fused_max_one_wave : ctx->fused_max_multi;   // one wave of CTAs or not
    p.fused = !(flags & DRA_F_NODE_SORTED) && !(ctx->cfg_flags & DRA_CFG_NO_FUSED) && n_claim <= fused_max_claims &&
              (uint64_t)n_node * n_claim <= ctx->fused_max_work && p.smem <= 225 * 1024 && n_node <= 16384;
    return p;
}

// CTAs of k_fused<FUSED_NW, stage> that can be resident at once with smem bytes of dynamic shared memory (the last
// answer is cached)
int fused_resident_ctas(dra_ctx* ctx, bool stage, size_t smem, int& ctas) {
    if (ctx->fused_occ_stage != (int)stage || ctx->fused_occ_smem != (int)smem) {
        int nb = 0;
        if (stage) CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_fused<FUSED_NW, true>, FUSED_NW * 32, smem));
        else CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_fused<FUSED_NW, false>, FUSED_NW * 32, smem));
        ctx->fused_occ_stage = (int)stage; ctx->fused_occ_smem = (int)smem; ctx->fused_occ_cta = nb * ctx->n_sm;
    }
    ctas = ctx->fused_occ_cta;
    return DRA_OK;
}

// The counting sort's widest node range: its one-warp histogram (the form for ranges too wide for the CTA-wide one)
// keeps (n_node + 1) u16 counters in shared memory, at most SORT_SMEM_MAX bytes of them
constexpr size_t SORT_SMEM_MAX = 200 * 1024;
size_t sort_warp_hist_smem(uint32_t n_node) { return ((size_t)n_node + 1) * sizeof(uint16_t); }

// Stable counting sort of 16-byte records by their node key (.y) into ctx->d_sorted + ctx->d_claim_off — the
// front half of the sort path.  Records naming no node get an INVALID OutRec (d_out != nullptr) or are dropped
// (d_out == nullptr: pod records).  Enqueues only.
int launch_sort(dra_ctx* ctx, const uint4* d_claims, uint32_t n_claim, const uint32_t* d_out_off, uint2* d_out,
                uint32_t n_out, uint32_t flags, Prof& prof, const void* inv_src, LaunchAttr pdl,
                uint32_t n_node, const uint32_t* d_node_off, const uint32_t* n_dev = nullptr) {
    Err err = err_of(ctx);
    // sort path: the kernels after the first are launched with pdl (pdl_attr, or LA_NONE)
    if (flags & DRA_F_NODE_SORTED) {
        if (n_dev) return fail(ctx, DRA_E_INVAL, "DRA_F_NODE_SORTED is not supported by the sharded call");
        uint32_t blocks = std::max(1u, (n_claim + 255) / 256);
        k_sorted_prep<<<blocks, 256, 0, ctx->stream>>>(d_claims, n_claim, n_node, d_out_off, ctx->d_claim_off,
                                                       ctx->d_sorted, d_out, n_out, err);
        ctx->launches += 1; ctx->chain |= DRA_K_SORTED_PREP;
        prof.mark(); prof.skip_to(3);
    } else {
        const size_t nbp = ((size_t)n_node + 2) & ~(size_t)1;
        const size_t small_smem = nbp * 4 + 32 * nbp * 2 + (size_t)n_claim * 2 + 16;
        if (n_claim <= 8192 && small_smem <= 200 * 1024) {
            // one launch: the whole stable counting sort in a single CTA
            Prefetch pf;
            pf.p[0] = inv_src;
            pf.bytes[0] = std::min<uint32_t>(ctx->n_gpu * 16u, 1u << 20) & ~15u;
            pf.p[1] = (const void*)((uintptr_t)d_node_off & ~(uintptr_t)15);      // (a shard's view starts mid-array: bulk prefetch wants 16-byte alignment)
            pf.bytes[1] = std::min<uint32_t>((n_node + 1) * 4u, 1u << 20) & ~15u;
            pf.p[2] = ctx->d_tbl; pf.bytes[2] = 1024;
            k_bucket_small<<<1, 1024, small_smem, ctx->stream>>>(d_claims, n_claim, n_node, d_out_off, ctx->d_claim_off,
                                                                 ctx->d_sorted, d_out, n_out, err, pf, n_dev);
            ctx->launches += 1; ctx->chain |= DRA_K_BUCKET_SMALL;
            prof.mark(); prof.skip_to(3);
        } else {
            Tiling t = tiling(n_claim, n_node, ctx->n_sm);
            if (t.cta_wide) {
                const size_t smem = (size_t)8 * (((size_t)n_node + 2) & ~(size_t)1) * 2;
                if (t.T == H8_TILE) k_bucket_hist8<false><<<t.n_tiles, 256, smem, ctx->stream>>>(d_claims, n_claim, n_node, ctx->d_hist, ctx->d_rank, n_dev, t.T);
                else k_bucket_hist8<true><<<t.n_tiles, 256, smem, ctx->stream>>>(d_claims, n_claim, n_node, ctx->d_hist, ctx->d_rank, n_dev, t.T);
                ctx->chain |= t.T == H8_TILE ? DRA_K_HIST8 : DRA_K_HIST8_MULTI;
                prof.mark();
                // the scan: a warp per node with every load in flight at once (latency), or — big matrices — coalesced rows
                if ((size_t)t.n_tiles * (n_node + 1) > (size_t)512 * 1024) {
                    const uint32_t n_cta = (n_node + 1 + 31) / 32;
                    if (ctx->cap_scan_status < n_cta) return fail(ctx, DRA_E_STATE, "scan status words not allocated (ensure_batch)");
                    CU(launch_k(k_bucket_scan_rows, dim3(n_cta), dim3(256), 0, ctx->stream, pdl, ctx->d_hist, t.n_tiles, n_node, ctx->d_claim_off, ctx->d_ticket + TK_SCAN_ROWS, ctx->d_scan_status, err));
                    ctx->chain |= DRA_K_SCAN_ROWS;
                } else {
                    CU(launch_k(k_bucket_scan8, dim3((n_node + 1 + 7) / 8), dim3(256), 0, ctx->stream, pdl, ctx->d_hist, t.n_tiles, n_node, ctx->d_claim_off, ctx->d_ticket + TK_SCAN8));
                    ctx->chain |= DRA_K_SCAN8;
                }
                prof.mark();
            } else {
                if (n_dev) return fail(ctx, DRA_E_INVAL, "sharded call: node range too wide for the CTA-wide histogram");
                size_t smem = sort_warp_hist_smem(n_node);
                if (smem > SORT_SMEM_MAX) return fail(ctx, DRA_E_INVAL, "n_node=%u exceeds the bucketing limit", n_node);
                k_bucket_hist<<<t.n_tiles, 32, smem, ctx->stream>>>(d_claims, n_claim, n_node, t.T, ctx->d_hist, ctx->d_rank);
                prof.mark();
                CU(launch_k(k_bucket_scan, dim3(1), dim3(1024), 0, ctx->stream, pdl, ctx->d_hist, t.n_tiles, n_node, ctx->d_claim_off));
                ctx->chain |= DRA_K_HIST_WARP | DRA_K_SCAN;
                prof.mark();
            }
            uint32_t blocks = std::max(1u, (n_claim + 255) / 256);
            CU(launch_k(k_bucket_scatter, dim3(blocks), dim3(256), 0, ctx->stream, pdl, d_claims, n_claim, n_node, t.T, ctx->d_hist, ctx->d_rank,
                        ctx->d_claim_off, d_out_off, ctx->d_sorted, d_out, n_out, err, n_dev));
            prof.mark();
            ctx->launches += 3; ctx->chain |= DRA_K_SCATTER; ctx->chain_tile = t.T;
        }
    }

    return DRA_OK;
}

// The part of the inventory a launch works on (sharded call: this rank's node range; claims carry LOCAL node
// indices, GPU indices stay global because node_off keeps its global values) and where the claim count comes from.
struct AllocView {
    uint32_t node_lo = 0, n_node = 0;
    const uint32_t* n_dev = nullptr;      // device-side claim count (the claim list was compacted on the device)
    int have_off = -1;                    // -1: from d_out_off; else the CALLER's out_off convention (spec §1/§3)
    const ShardArgs* sa = nullptr;        // the compaction that produces the claim list, launched by launch_allocate
    uint32_t sc_rows = 1; bool sc_flat = true;
};

int launch_compaction(dra_ctx* ctx, const ShardArgs& sa, uint32_t sc_rows, bool sc_flat) {
    if (!sc_flat) k_shard_compact<<<sa.n_tiles, 256, 0, ctx->stream>>>(sa);
    else if (sc_rows == 1) k_shard_compact_flat<1><<<sa.n_tiles, 256, 0, ctx->stream>>>(sa);
    else k_shard_compact_flat<8><<<sa.n_tiles, 256, 0, ctx->stream>>>(sa);
    ctx->launches += 1;
    ctx->chain |= !sc_flat ? DRA_K_COMPACT_LOOKBACK : sc_rows == 1 ? DRA_K_COMPACT_FLAT1 : DRA_K_COMPACT_FLAT8;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "shard compaction launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int launch_allocate(dra_ctx* ctx, const uint4* d_claims, uint32_t n_claim, const uint32_t* d_out_off,
                    uint2* d_out, uint32_t n_out, uint32_t flags, const PktGather* tail = nullptr, bool* tail_done = nullptr,
                    const AllocView* view = nullptr) {
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    int rc = upload_table(ctx);
    if (rc) return rc;
    const uint32_t n_node = view ? view->n_node : ctx->n_node;
    const uint32_t* d_node_off = ctx->d_node_off + (view ? view->node_lo : 0u);
    const uint32_t* n_dev = view ? view->n_dev : nullptr;
    Err err = err_of(ctx);
    Prof prof(ctx);
    if (view && view->sa && (rc = launch_compaction(ctx, *view->sa, view->sc_rows, view->sc_flat))) return rc;

    PackArgs a;
    memset(&a, 0, sizeof a);
    a.inv_src = (flags & DRA_F_FRESH_INVENTORY) ? ctx->d_inv_pristine : ctx->d_inv_live;
    a.inv_dst = ctx->d_inv_live;
    a.node_off = d_node_off;
    a.tbl = ctx->d_tbl;
    a.out = d_out; a.n_out = n_out; a.n_node = n_node;
    a.have_off = (view && view->have_off >= 0) ? (uint32_t)view->have_off : (d_out_off != nullptr);
    a.n_dev = n_dev;
    a.err = err;
    a.sel = sel_of(ctx);

    const FusedPlan plan = fused_plan(ctx, n_claim, flags, n_node);
    const bool fused = plan.fused, stage = plan.stage;
    const size_t fused_smem = plan.smem;
    const DirectIO dio = ctx->dio_pending;
    ctx->dio_pending = DirectIO{};
    if (dio.h_claims && !(fused && stage)) return fail(ctx, DRA_E_STATE, "direct host I/O was planned for a batch that does not take the staged single-launch kernel");
    if (fused) {
        // the gather tail has every CTA wait for its peers' packets: all CTAs of the grid must be resident at once.
        // Shared memory left over goes to the send queue (records leave for the peers while the pack still runs).
        size_t launch_smem = fused_smem;
        if (tail) {
            const size_t room = fused_smem + 32 <= 225 * 1024 ? (225 * 1024 - fused_smem - 32) / 16 : 0;
            const uint32_t q_cap = (uint32_t)std::min<size_t>(room, 2048);
            const size_t tail_smem = fused_smem + 32 + (size_t)q_cap * 16;
            int ctas = 0;
            if ((rc = fused_resident_ctas(ctx, stage, tail_smem, ctas))) return rc;
            if ((int)(n_node + 1) <= ctas) { a.peer = *tail; a.q_cap = q_cap; launch_smem = tail_smem; if (tail_done) *tail_done = true; }
        }
        a.claims = d_claims; a.out_off = d_out_off; a.n_claim = n_claim;
        if (getenv("DRA_TIMELINE")) {           // instrumentation only: per-CTA clock stamps of the last fused launch
            if (ctx->tl_cap < (size_t)(2 * n_node + 24) * 8) {
                if (ctx->d_timeline) CU(cudaFree(ctx->d_timeline));
                ctx->tl_cap = (size_t)(2 * n_node + 24) * 8 + 64;
                CU(cudaMalloc((void**)&ctx->d_timeline, ctx->tl_cap * 8));
                CU(cudaMemsetAsync(ctx->d_timeline, 0, ctx->tl_cap * 8, ctx->stream));     // (only here: a memset between the kernels of a step would sit on the measured path)
            }
            a.timeline = ctx->d_timeline; ctx->tl_n = (2 * n_node + 6) * 8;
        }
        prof.skip_to(3);
        // grid = one CTA per node + one CTA for the claims that name no node
        const dim3 grid(n_node + 1), block(FUSED_NW * 32);
        if (stage && dio.h_claims) {
            // direct host I/O: two grid barriers inside, so every CTA must be resident — cooperative launch
            a.dio = dio;
            CU(launch_k(k_fused<FUSED_NW, true>, grid, block, fused_smem, ctx->stream, LA_COOP, a));
        } else {
            const LaunchAttr dep = n_dev ? pdl_attr(ctx) : LA_NONE;      // programmatic dependent of the compaction
            if (stage) CU(launch_k(k_fused<FUSED_NW, true>, grid, block, launch_smem, ctx->stream, dep, a));
            else CU(launch_k(k_fused<FUSED_NW, false>, grid, block, launch_smem, ctx->stream, dep, a));
        }
        ctx->launches += 1;
        ctx->chain |= (stage && dio.h_claims) ? DRA_K_FUSED_DIRECT : stage ? DRA_K_FUSED_STAGED : DRA_K_FUSED_STREAM;
        prof.mark();
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "kernel launch: %s", cudaGetErrorString(e));
        return DRA_OK;
    }

    const LaunchAttr pdl = pdl_attr(ctx);
    if ((rc = launch_sort(ctx, d_claims, n_claim, d_out_off, d_out, n_out, flags, prof, a.inv_src, pdl, n_node, d_node_off, n_dev))) return rc;

    a.sorted = ctx->d_sorted;
    a.claim_off = ctx->d_claim_off;
    if (n_node) {
        if (n_node <= (uint32_t)ctx->n_sm * 16u) {
            CU(launch_k(k_pack<1>, dim3(n_node), dim3(32), pack_smem_bytes(1), ctx->stream, pdl, a));
            ctx->chain |= DRA_K_PACK1;
        } else {
            // more nodes than warps can be resident: CTAs of 4 warps, exactly as many as fit at once, each warp walking nodes
            if (ctx->pack4_occ < 0) {
                int nb = 0;
                CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_pack<4>, 128, pack_smem_bytes(4)));
                ctx->pack4_occ = std::max(1, nb);
            }
            CU(launch_k(k_pack<4>, dim3(std::min((n_node + 3) / 4, (uint32_t)(ctx->n_sm * ctx->pack4_occ))), dim3(128), pack_smem_bytes(4), ctx->stream, pdl, a));
            ctx->chain |= DRA_K_PACK4;
        }
        ctx->launches += 1;
    }
    prof.mark();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "kernel launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

// Lanes per (pod, node) pair for the pair kernels (k_unsuitable, preemption's, pod capacity's): one per GPU of the widest node
uint32_t pair_width(const dra_ctx* ctx) { return ctx->max_width <= 8 ? 8u : (ctx->max_width <= 16 ? 16u : 32u); }

// f(std::integral_constant<int, W>{}) for W = pair_width: f launches the pair kernel instantiated for W
template <class F>
void at_pair_width(const dra_ctx* ctx, F&& f) {
    const uint32_t W = pair_width(ctx);
    if (W == 8) f(std::integral_constant<int, 8>{});
    else if (W == 16) f(std::integral_constant<int, 16>{});
    else f(std::integral_constant<int, 32>{});
}

// A pair kernel's grid for n pairs (or pods): 8 warps of 32 / W pairs per CTA, at most 8 CTAs per SM
uint32_t pair_grid(const dra_ctx* ctx, uint32_t n) {
    const uint32_t per_cta = 8 * (32 / pair_width(ctx));
    return std::max(1u, std::min((n + per_cta - 1) / per_cta, (uint32_t)ctx->n_sm * 8u));
}

// k_unsuitable over a.n_walk pairs (win: the sharded call's node window and gate; else the whole inventory; why: the
// reasons of spec §17 into a.why / a.why_claim instead of the bits, at the walk index).  Enqueues only.
int launch_unsuitable(dra_ctx* ctx, UnsArgs& a, bool win, bool why = false) {
    const uint32_t grid = pair_grid(ctx, a.n_walk);
    if (a.exhaustive) { if (int rc = walk_counter(ctx, TK_WALK_UNSUITABLE, a.work)) return rc; }
    at_pair_width(ctx, [&](auto w) {
        constexpr int W = decltype(w)::value;
        const auto k = why ? (win ? (a.exhaustive ? k_unsuitable<8, W, true, true, true> : k_unsuitable<8, W, false, true, true>)
                                  : (a.exhaustive ? k_unsuitable<8, W, true, false, true> : k_unsuitable<8, W, false, false, true>))
                     : win ? (a.exhaustive ? k_unsuitable<8, W, true, true> : k_unsuitable<8, W, false, true>)
                           : (a.exhaustive ? k_unsuitable<8, W, true, false> : k_unsuitable<8, W, false, false>);
        k<<<grid, 256, 0, ctx->stream>>>(a);
    });
    ctx->launches += 1;
    return DRA_OK;
}

int collect_timings(dra_ctx* ctx, int n_marks) {
    if (!ctx->profiling) return DRA_OK;
    for (int i = 0; i < 5; ++i) ctx->timings[i] = 0.f;
    for (int i = 0; i < n_marks && i < 5; ++i) {
        float ms = 0.f;
        if (!((ctx->ev_mask >> i) & 1u) || !((ctx->ev_mask >> (i + 1)) & 1u)) continue;
        if (cudaEventElapsedTime(&ms, ctx->ev[i], ctx->ev[i + 1]) == cudaSuccess) ctx->timings[i] = ms * 1000.f;
    }
    (void)cudaGetLastError();   // an event that was never recorded is not an error of the batch
    return DRA_OK;
}

int check_err(dra_ctx* ctx) {
    uint32_t oor = ctx->h_err[ERR_OUT_RANGE], ns = ctx->h_err[ERR_NOT_SORTED], pt = ctx->h_err[ERR_PEER_TIMEOUT], sp = ctx->h_err[ERR_SHARD_PLAN];
    const uint32_t dw = ctx->h_err[ERR_DEVICE_WAIT], bo = ctx->h_err[ERR_BAD_OFFSETS], bp = ctx->h_err[ERR_BAD_PODS];
    const uint32_t bd = ctx->h_err[ERR_BAD_DEALLOC];
    if (!oor && !ns && !pt && !sp && !dw && !bo && !bp && !bd) return DRA_OK;
    for (uint32_t i = 0; i < ERR_WORDS; ++i) ctx->h_err[i] = 0;
    cudaMemsetAsync(ctx->d_err, 0, ERR_WORDS * sizeof(uint32_t), ctx->stream);
    cudaStreamSynchronize(ctx->stream);
    if (sp) return fail(ctx, DRA_E_STATE, "sharded call: %u claims fell into this shard, more than the launch was laid out for; nothing was changed, call again", ctx->h_sc_counts ? ctx->h_sc_counts[0] : 0u);
    if (dw && (ctx->chain & DRA_K_PREEMPT_PLACE_SHARD))
        return fail(ctx, DRA_E_CUDA, "sharded preempt and place: the walk's wait timed out (its CTAs were not resident together); nothing was "
                                     "written: no output, and every inventory is as it was");
    if (dw) return fail(ctx, DRA_E_CUDA, "a device-side wait inside one kernel (grid barrier / look-back over CTAs) timed out: CTAs were not scheduled together; state is undefined, reload the inventory");
    if (bo && (ctx->chain & DRA_K_PREEMPT_PLACE))
        return fail(ctx, DRA_E_INVAL, "dra_preempt_place_batch: running pods: pod_off not monotone or not spanning the claims, a slot range "
                                      "outside n_out, or OK slots naming a GPU index >= n_gpu or GPUs of two nodes; nothing was written");
    if (bo && (ctx->chain & DRA_K_PREEMPT))
        return fail(ctx, DRA_E_INVAL, "dra_preempt_batch: running pods: pod_off not monotone or not spanning the claims, a slot range outside "
                                      "n_out, OK slots naming a GPU index >= n_gpu or GPUs of two nodes, or a budget neither "
                                      "DRA_PDB_NONE nor below n_pdb; nothing was written");
    if (bo && (ctx->chain & DRA_K_PREEMPT_SHARD))
        return fail(ctx, DRA_E_INVAL, "sharded preemption: pod_off / cand_off not monotone or not spanning their arrays, or running pods: pod_off "
                                      "not monotone or not spanning the claims, a slot range outside n_out, OK slots naming a GPU index "
                                      ">= n_gpu or GPUs of two nodes, or a budget neither DRA_PDB_NONE nor below n_pdb (on this rank "
                                      "or a peer); nothing was written");
    if (bo && (ctx->chain & DRA_K_PREEMPT_PLACE_SHARD))
        return fail(ctx, DRA_E_INVAL, "sharded preempt and place: pod_off / cand_off not monotone or not spanning their arrays, more than %u "
                                      "candidates for a pod, a pending slot outside n_out, or running pods: pod_off not monotone or not "
                                      "spanning the claims, a slot range outside n_out, or OK slots naming a GPU index >= n_gpu or GPUs of "
                                      "two nodes; nothing was written", PL_POS);
    if (bo && (ctx->chain & DRA_K_UNSUITABLE_WHY_SHARD))
        return fail(ctx, DRA_E_INVAL, "sharded unsuitable reasons: pod_off / cand_off not monotone or not spanning their arrays (on this "
                                      "rank or a peer); nothing was written");
    if (bo) return fail(ctx, DRA_E_INVAL, "sharded UnsuitableNodes: pod_off / cand_off not monotone or not spanning their arrays; nothing was evaluated");
    if (bp && (ctx->chain & DRA_K_PLACE_SHARD))
        return fail(ctx, DRA_E_INVAL, "sharded place pods: pod_off / cand_off not monotone or not spanning their arrays, more than %u candidates for a pod, "
                                      "a pod's OutRec slots outside n_out, or one rank's slots beyond the cap_per_rank of dra_shard_export; "
                                      "no inventory was changed", PL_POS);
    if (bp) return fail(ctx, DRA_E_INVAL, "sharded pods Allocate: pod_off not monotone or not spanning [0, n_claim], a pod's OutRec slots outside n_out, "
                                          "or one rank's slots beyond the cap_per_rank of dra_shard_export; no inventory was changed");
    if (bd) return fail(ctx, DRA_E_INVAL, "sharded Deallocate: out_off/n_out: a claim's slots fall outside out[]; no record was applied, inventory unchanged");
    if (pt) return fail(ctx, DRA_E_NCCL, "all-gather: a rank did not deliver its records in time (or aborted its batch)");
    if (ns) return fail(ctx, DRA_E_INVAL, "DRA_F_NODE_SORTED given but claims are not sorted by node; inventory unchanged");
    return fail(ctx, DRA_E_INVAL, "out_off/n_out: a claim's slots fall outside out[]; inventory state is undefined, reset it");
}

// The device buffers of a §15 walk (dra_preempt_place_batch and its sharded form) for n_pod pending pods, n_pair judged
// pairs (n_pod * n_node in the dense form) and rn_pod running pods
int pp_buffers(dra_ctx* ctx, uint32_t n_pod, uint32_t n_pair, uint32_t rn_pod) {
    const size_t pods = (size_t)n_pod + 8, pairs = (size_t)n_pair + 8, rpods = (size_t)rn_pod + 8, nodes = (size_t)ctx->n_node + 8;
    int rc;
    if ((rc = grow_set(ctx, ctx->cap_podrec, pairs, ctx->d_podrec)) ||
        (rc = grow_set(ctx, ctx->cap_place_pods, pods, ctx->d_place_state, ctx->d_place_node)) ||
        (rc = grow_set(ctx, ctx->cap_place_cursor, nodes, ctx->d_place_cursor)) ||
        (rc = grow_set(ctx, ctx->cap_pre_pods, pods, ctx->d_pre_prio, ctx->d_pre_node, ctx->d_pre_nvic, ctx->d_pre_choice, ctx->d_pre_pst,
                       ctx->d_pre_podviol)) ||
        (rc = grow_set(ctx, ctx->cap_pre_pairs, pairs, ctx->d_pre_psum, ctx->d_pre_psum64, ctx->d_pre_pairst, ctx->d_pre_pairvic,
                       ctx->d_pre_pairviol)) ||
        (rc = grow_set(ctx, ctx->cap_pre_rpods, rpods, ctx->d_pre_rpodoff, ctx->d_pre_rprio, ctx->d_pre_rrec, ctx->d_pre_vlist,
                       ctx->d_pre_rpdb, ctx->d_pre_vprev)) ||
        (rc = grow_set(ctx, ctx->cap_pp_pods, pods, ctx->d_pp_pending)) ||
        (rc = grow_set(ctx, ctx->cap_pp_rpods, rpods, ctx->d_pp_evicted)) ||
        (rc = grow_set(ctx, ctx->cap_pp_nodes, nodes, ctx->d_pp_runoff, ctx->d_pp_judged))) return rc;
    return DRA_OK;
}

size_t al16(size_t b) { return (b + 15) & ~(size_t)15; }

// The inputs of a synchronous call, each part from the host at src to the device at dst.  A part without src is written
// by the caller (stage_in's fill).  A fixed array, nothing allocated per call: a part beyond CAP is not kept, and
// stage_in refuses the call.
struct Staging {
    static constexpr int CAP = 14;
    struct Part { void* dst; const void* src; size_t bytes; };
    Part part[CAP];
    int n = 0;
    bool overflow = false;
    void add(void* dst, const void* src, size_t bytes) {
        if (n < CAP) part[n++] = Part{dst, src, bytes};
        else overflow = true;
    }
};

// s's parts through the pinned h_in (grown once), each at a 16-byte boundary; parts of no bytes are skipped.  Each part is
// copied in, or for the part without src written by fill(its staging), before its copy to the device is enqueued.
template <class Fill>
int stage_in(dra_ctx* ctx, const Staging& s, Fill fill) {
    if (s.overflow) return fail(ctx, DRA_E_STATE, "more than %d staged inputs in one call", Staging::CAP);
    size_t total = 0;
    for (int i = 0; i < s.n; ++i) total += al16(s.part[i].bytes);
    if (int rc = grow_pinned(ctx, ctx->h_in, ctx->h_in_cap, total)) return rc;
    uint8_t* h = ctx->h_in;
    for (int i = 0; i < s.n; ++i) {
        const Staging::Part& p = s.part[i];
        if (!p.bytes) continue;
        if (p.src) memcpy(h, p.src, p.bytes);
        else fill(h);
        CU(cudaMemcpyAsync(p.dst, h, p.bytes, cudaMemcpyHostToDevice, ctx->stream));
        h += al16(p.bytes);
    }
    return DRA_OK;
}
int stage_in(dra_ctx* ctx, const Staging& s) { return stage_in(ctx, s, [](uint8_t*) {}); }

// The caller's running pods R as parts of s, into the d_pre_r* buffers (grown as needed); dev = R with those device pointers.
// B (NULL: none): the budgets too, Bd = B with device pointers.
int running_parts(dra_ctx* ctx, const dra_running_pods& R, Staging& s, dra_running_pods& dev,
                  const dra_disruption_budgets* B = nullptr, dra_disruption_budgets* Bd = nullptr) {
    int rc;
    if ((rc = grow_set(ctx, ctx->cap_pre_rclaims, (size_t)R.n_claim + 8, ctx->d_pre_rclaims, ctx->d_pre_routoff)) ||
        (rc = grow_set(ctx, ctx->cap_pre_rpods, (size_t)R.n_pod + 8, ctx->d_pre_rpodoff, ctx->d_pre_rprio, ctx->d_pre_rrec, ctx->d_pre_vlist,
                       ctx->d_pre_rpdb, ctx->d_pre_vprev)) ||
        (rc = grow_set(ctx, ctx->cap_pre_rout, (size_t)R.n_out + 8, ctx->d_pre_rout))) return rc;
    s.add(ctx->d_pre_rclaims, R.claims, (size_t)R.n_claim * 16);
    s.add(ctx->d_pre_rpodoff, R.pod_off, ((size_t)R.n_pod + 1) * 4);
    s.add(ctx->d_pre_rprio, R.prio, (size_t)R.n_pod * 4);
    s.add(ctx->d_pre_routoff, R.out_off, R.out_off ? (size_t)R.n_claim * 4 : 0);
    s.add(ctx->d_pre_rout, R.out, (size_t)R.n_out * 8);
    dev = R;
    dev.claims = (const dra_claim_rec*)ctx->d_pre_rclaims; dev.pod_off = ctx->d_pre_rpodoff;
    dev.prio = (const int32_t*)ctx->d_pre_rprio; dev.out_off = R.out_off ? ctx->d_pre_routoff : nullptr;
    dev.out = (const dra_out_rec*)ctx->d_pre_rout;
    if (!B) return DRA_OK;
    if ((rc = grow_set(ctx, ctx->cap_pre_allowed, (size_t)B->n_pdb + 8, ctx->d_pre_allowed))) return rc;
    s.add(ctx->d_pre_rpdb, B->run_pdb, B->run_pdb ? (size_t)R.n_pod * 4 : 0);
    s.add(ctx->d_pre_allowed, B->allowed, B->n_pdb ? (size_t)B->n_pdb * 4 : 0);
    *Bd = *B;
    Bd->run_pdb = B->run_pdb ? ctx->d_pre_rpdb : nullptr; Bd->allowed = B->n_pdb ? ctx->d_pre_allowed : nullptr;
    return DRA_OK;
}

// pair -> pod of the candidate form: pair_pod[k] = q for every k in [cand_off[q], cand_off[q + 1])
void expand_pairs(uint32_t* pair_pod, const uint32_t* cand_off, uint32_t n_pod) {
    for (uint32_t q = 0; q < n_pod; ++q)
        for (uint32_t k = cand_off[q]; k < cand_off[q + 1]; ++k) pair_pod[k] = q;
}

// One output of a synchronous call: bytes from the device at src to the caller's dst
struct ReadBack { void* dst; const void* src; size_t bytes; };

// The outputs of a synchronous call.  A fixed array like Staging: an output beyond CAP is not kept, and reserve_out
// refuses the call.
struct Outputs {
    static constexpr int CAP = 12;
    ReadBack out[CAP];
    int n = 0;
    bool overflow = false;
    Outputs(std::initializer_list<ReadBack> l = {}) { for (const ReadBack& o : l) add(o.dst, o.src, o.bytes); }
    void add(void* dst, const void* src, size_t bytes) {
        if (n < CAP) out[n++] = ReadBack{dst, src, bytes};
        else overflow = true;
    }
    const ReadBack* begin() const { return out; }
    const ReadBack* end() const { return out + n; }
    size_t bytes() const { size_t t = 0; for (const ReadBack& o : *this) t += al16(o.bytes); return t; }
};

// The pinned h_out for outs, grown before the call enqueues anything: a failed allocation leaves the inventory as it was
int reserve_out(dra_ctx* ctx, const Outputs& outs) {
    if (outs.overflow) return fail(ctx, DRA_E_STATE, "more than %d outputs in one call", Outputs::CAP);
    return grow_pinned(ctx, ctx->h_out, ctx->h_out_cap, outs.bytes());
}

// The tail of a synchronous call: the outputs into h_out (reserve_out), one synchronise, the launch error as DRA_E_CUDA
// "<name>: ...", the times of n_marks stages, the device's fault words; the caller's buffers are written only when all passed
int read_back(dra_ctx* ctx, const char* name, int n_marks, const Outputs& outs) {
    if (outs.bytes() > ctx->h_out_cap) return fail(ctx, DRA_E_STATE, "%s: outputs not reserved before the launch", name);
    uint8_t* h = ctx->h_out;
    for (const ReadBack& o : outs) {
        if (o.bytes) CU(cudaMemcpyAsync(h, o.src, o.bytes, cudaMemcpyDeviceToHost, ctx->stream));
        h += al16(o.bytes);
    }
    CU(cudaStreamSynchronize(ctx->stream));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "%s: %s", name, cudaGetErrorString(e));
    collect_timings(ctx, n_marks);
    if (int rc = check_err(ctx)) return rc;
    h = ctx->h_out;
    for (const ReadBack& o : outs) {
        if (o.bytes) memcpy(o.dst, h, o.bytes);
        h += al16(o.bytes);
    }
    return DRA_OK;
}

// The pending pods' pod_off [n_pod + 1]: spans [0, n_claim] and is monotone
int check_pod_off(dra_ctx* ctx, const uint32_t* pod_off, uint32_t n_pod, uint32_t n_claim) {
    if (pod_off[0] != 0 || pod_off[n_pod] != n_claim) return fail(ctx, DRA_E_INVAL, "pod_off must span [0, n_claim]");
    for (uint32_t q = 0; q < n_pod; ++q)
        if (pod_off[q + 1] < pod_off[q]) return fail(ctx, DRA_E_INVAL, "pod_off not monotone at pod %u", q);
    return DRA_OK;
}

// The pending pods' candidates: the dense form (cand_nodes and cand_off both NULL: every pod against every node), or
// cand_off [n_pod + 1] from 0 and monotone with at most per_pod candidates a pod, and cand_nodes when it lists any.
// n_pair: the pairs, n_pod * dense_nodes in the dense form; more than max_pairs fails.
int check_cands(dra_ctx* ctx, uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t per_pod,
                uint32_t dense_nodes, uint64_t max_pairs, bool& dense, uint32_t& n_pair) {
    dense = cand_nodes == nullptr && cand_off == nullptr;
    if (!dense && !cand_off) return fail(ctx, DRA_E_INVAL, "cand_nodes without cand_off");
    if (!dense && cand_off[0] != 0) return fail(ctx, DRA_E_INVAL, "cand_off[0] must be 0");
    for (uint32_t q = 0; !dense && q < n_pod; ++q) {
        if (cand_off[q + 1] < cand_off[q]) return fail(ctx, DRA_E_INVAL, "cand_off not monotone at pod %u", q);
        if (cand_off[q + 1] - cand_off[q] > per_pod) return fail(ctx, DRA_E_INVAL, "pod %u has more than %u candidates", q, per_pod);
    }
    const uint64_t n = dense ? (uint64_t)n_pod * dense_nodes : cand_off[n_pod];
    if (n > max_pairs) return fail(ctx, DRA_E_INVAL, "%llu (pod, node) pairs: more than %llu", (unsigned long long)n, (unsigned long long)max_pairs);
    n_pair = (uint32_t)n;
    if (n_pair && !dense && !cand_nodes) return fail(ctx, DRA_E_INVAL, "cand_off lists candidates but cand_nodes is NULL");
    return DRA_OK;
}

// The slots of the pod calls and dra_deallocate_batch: n_out >= n_claim without out_off, and each claim's OutRec slots
// within n_out.  A GPU claim of count 1 .. DRA_MAX_COUNT (more than 1 only with out_off) has count slots, every other
// claim one.  any_node (spec §13): counted as if the claim named a node of the inventory; otherwise (spec §12, as
// k_pod_records and k_dealloc count them) only a GPU claim naming a node < n_node has count slots.
int check_slots(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* out_off, uint32_t n_out,
                bool any_node) {
    if (!out_off) {                                       // one slot per claim: claim i owns slot i
        if (n_out < n_claim) return fail(ctx, DRA_E_INVAL, "n_out %u < n_claim %u without out_off", n_out, n_claim);
        return DRA_OK;
    }
    for (uint32_t i = 0; i < n_claim; ++i) {
        const dra_claim_rec& c = claims[i];
        const bool gpu = c.kind == DRA_KIND_GPU && (any_node || c.node < ctx->n_node) && c.count >= 1 && c.count <= DRA_MAX_COUNT;
        const uint32_t slots = gpu ? c.count : 1u, dst = out_off[i];
        if (dst > n_out || slots > n_out - dst) return fail(ctx, DRA_E_INVAL, "claim %u: slots [%u, %u) outside n_out %u", i, dst, dst + slots, n_out);
    }
    return DRA_OK;
}

// A call that will sort n_rec records (pod or pair records, running pods) by node over the whole inventory: a node range
// wider than the counting sort takes (launch_sort) fails here, before anything is staged or launched, so the refusal
// leaves no kernel behind and no fault word set for the next call
int check_sortable(dra_ctx* ctx, uint32_t n_rec) {
    if (n_rec && sort_warp_hist_smem(ctx->n_node) > SORT_SMEM_MAX)
        return fail(ctx, DRA_E_INVAL, "n_node=%u exceeds the bucketing limit", ctx->n_node);
    return DRA_OK;
}

// occ: how many CTAs of 4 warps of the walk k can be resident per SM, queried once; none fails
template <class K>
int walk_occupancy(dra_ctx* ctx, int& occ, const char* name, K k) {
    if (occ < 0) {
        int nb = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k, 128, 0));
        occ = nb;
    }
    if (occ < 1) return fail(ctx, DRA_E_CUDA, "%s: no CTA can be resident", name);
    return DRA_OK;
}

// A persistent walk k over the inventory's nodes (none: no launch): CTAs of 4 warps, one per 4 nodes up to all that can be
// resident at once (walk_occupancy), launched cooperatively so that every one of them is.  Enqueues only.
template <typename... KA, typename... A>
int launch_walk(dra_ctx* ctx, int& occ, const char* name, void (*k)(KA...), A&&... args) {
    if (!ctx->n_node) return DRA_OK;
    if (int rc = walk_occupancy(ctx, occ, name, k)) return rc;
    const uint32_t grid = std::max(1u, std::min((ctx->n_node + 3) / 4, (uint32_t)(occ * ctx->n_sm)));
    CU(launch_k(k, dim3(grid), dim3(128), 0, ctx->stream, LA_COOP, std::forward<A>(args)...));
    ctx->launches += 1;
    return DRA_OK;
}

// The grid of a sharded walk over n_walk nodes with every CTA resident (occ per SM).  Not a cooperative launch: ranks
// sharing this device run their walks side by side, so each takes its share of the residency, less one CTA per SM left
// for a peer's waiting kernel.
uint32_t shard_walk_grid(const dra_ctx* ctx, int occ, bool gather, uint32_t n_walk) {
    const int k = gather ? std::max(1, ctx->peers_on_device) : 1;
    const int per_sm = k > 1 ? std::max(1, occ - 1) : occ;
    const uint32_t share = (uint32_t)std::max(1, per_sm * ctx->n_sm / k);
    return std::max(1u, std::min((n_walk + 3) / 4, share));
}

// The PreArgs fields every preemption call sets: the pending pods (cand_nodes and cand_off nullptr in the dense form), the
// running pods R (device pointers), the running lists' buffers, the inventory copy inv that is judged, psum, the pod
// outputs and the fault gate
PreArgs pre_args(dra_ctx* ctx, const uint4* claims, const uint32_t* pod_off, const int32_t* prio, uint32_t n_pod,
                 const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t n_pair, const dra_running_pods& R,
                 const uint4* inv, uint32_t flags) {
    PreArgs a; memset(&a, 0, sizeof a);
    a.claims = claims; a.pod_off = pod_off; a.prio = prio; a.n_pod = n_pod;
    a.cand_nodes = cand_nodes; a.cand_off = cand_off; a.n_pair = n_pair;
    a.rclaims = (const uint4*)R.claims; a.rn_claim = R.n_claim; a.rpod_off = R.pod_off; a.rprio = R.prio; a.rn_pod = R.n_pod;
    a.rout_off = R.out_off; a.rout = (const uint2*)R.out; a.rn_out = R.n_out;
    a.rrec = ctx->d_pre_rrec; a.rsorted = ctx->d_sorted; a.list_off = ctx->d_claim_off; a.vlist = ctx->d_pre_vlist;
    a.inv = inv; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.n_gpu = ctx->n_gpu; a.tbl = ctx->d_tbl;
    a.sel = sel_of(ctx); a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u;
    a.psum = ctx->d_pre_psum; a.psum64 = ctx->d_pre_psum64;
    a.pod_node = ctx->d_pre_node; a.pod_status = ctx->d_pre_pst;
    a.gate = ctx->d_err + ERR_BAD_OFFSETS; a.err = err_of(ctx);
    return a;
}

// a's disruption budgets from B (pointers the device reads; NULL: none): run_pdb checked whenever given, the budgets in
// force when n_pdb > 0 and there are running pods
void pre_budgets(dra_ctx* ctx, PreArgs& a, const dra_disruption_budgets* B) {
    if (!B) return;
    a.run_pdb = a.rn_pod ? B->run_pdb : nullptr; a.pdb_allowed = B->allowed; a.n_pdb = B->n_pdb;
    a.pdb = B->n_pdb && a.rn_pod ? 1u : 0u;
    a.vprev = ctx->d_pre_vprev;
}

// The budget arguments of a preemption call that has pending pods (spec §14, "Disruption budgets"; NULL: none)
int check_budgets(dra_ctx* ctx, const char* name, const dra_disruption_budgets* B, uint32_t rn_pod) {
    if (!B || !B->n_pdb) return DRA_OK;
    if (!B->allowed) return fail(ctx, DRA_E_INVAL, "%s: n_pdb %u without allowed", name, B->n_pdb);
    if (rn_pod && !B->run_pdb) return fail(ctx, DRA_E_INVAL, "%s: %u running pods and %u budgets without run_pdb", name, rn_pod, B->n_pdb);
    if (rn_pod >= DRA_PDB_MAX_RUNNING)
        return fail(ctx, DRA_E_INVAL, "%s: %u running pods with budgets: at most %u", name, rn_pod, DRA_PDB_MAX_RUNNING - 1);
    return DRA_OK;
}

// The running lists: k_pre_running, its records bucketed by node with the counting sort (without running pods the
// offsets are zeroed instead) and k_pre_vsort.  walk (§15): the visit lists reuse the sort's buffers, so the offsets are
// kept in d_pp_runoff, which becomes a.list_off; and without running pods there is no list to sort.  Enqueues only.
int launch_running_lists(dra_ctx* ctx, PreArgs& a, Prof& prof, bool walk) {
    cudaStream_t st = ctx->stream;
    k_pre_running<<<std::max(1u, (a.rn_pod + 255) / 256), 256, 0, st>>>(a);
    ctx->launches += 1;
    if (!a.rn_pod) CU(cudaMemsetAsync(walk ? ctx->d_pp_runoff : ctx->d_claim_off, 0, ((size_t)ctx->n_node + 2) * 4, st));
    else if (int rc = launch_sort(ctx, a.rrec, a.rn_pod, nullptr, nullptr, 0, 0, prof, a.inv, LA_NONE, ctx->n_node, ctx->d_node_off))
        return rc;
    if (ctx->n_node && (a.rn_pod || !walk)) {
        k_pre_vsort<<<std::min(ctx->n_node, (uint32_t)ctx->n_sm * 8u), 256, 0, st>>>(a);
        ctx->launches += 1;
    }
    if (walk) {
        if (a.rn_pod) CU(cudaMemcpyAsync(ctx->d_pp_runoff, ctx->d_claim_off, ((size_t)ctx->n_node + 1) * 4, cudaMemcpyDeviceToDevice, st));
        a.list_off = ctx->d_pp_runoff;
    }
    return DRA_OK;
}

// k_pods_preempt over s's pairs (none: no launch).  Enqueues only.
int launch_preempt_pairs(dra_ctx* ctx, PreArgs a, const PreShard& s, bool why = false) {
    if (!s.n_walk) return DRA_OK;
    if (int rc = walk_counter(ctx, TK_WALK_PREEMPT, a.work)) return rc;
    const uint32_t grid = pair_grid(ctx, s.n_walk);
    if (why) at_pair_width(ctx, [&](auto w) { k_pods_preempt<8, decltype(w)::value, true><<<grid, 256, 0, ctx->stream>>>(a, s); });
    else at_pair_width(ctx, [&](auto w) { k_pods_preempt<8, decltype(w)::value><<<grid, 256, 0, ctx->stream>>>(a, s); });
    ctx->launches += 1;
    return DRA_OK;
}

// k_pods_preempt_victims for a's pods: pod p's chosen pair at choice[p * cstride], its row at rows + p * rstride.  Enqueues only.
void launch_preempt_victims(dra_ctx* ctx, const PreArgs& a, const uint32_t* choice, uint32_t cstride, uint32_t* rows, uint32_t rstride) {
    const uint32_t grid = pair_grid(ctx, a.n_pod);
    at_pair_width(ctx, [&](auto w) {
        k_pods_preempt_victims<8, decltype(w)::value><<<grid, 256, 0, ctx->stream>>>(a, choice, cstride, rows, rstride);
    });
    ctx->launches += 1;
}

// k_pods_capacity over a's walk (none: no launch), then k_pods_capacity_sum over its pods when a per-pod output is asked
// for.  Enqueues only.
int launch_capacity(dra_ctx* ctx, CapArgs a) {
    if (a.n_walk) {
        if (int rc = walk_counter(ctx, TK_WALK_CAPACITY, a.work)) return rc;
        const uint32_t grid = pair_grid(ctx, a.n_walk);
        at_pair_width(ctx, [&](auto w) { k_pods_capacity<8, decltype(w)::value><<<grid, 256, 0, ctx->stream>>>(a); });
        ctx->launches += 1;
    }
    if (a.pod_total || a.pod_nodes) {
        k_pods_capacity_sum<<<(a.n_pod + 7) / 8, 256, 0, ctx->stream>>>(a);
        ctx->launches += 1;
    }
    return DRA_OK;
}

// The caller's reason outputs of a reasons call (spec §17–§19): pair_why whenever there are pairs, the others when asked
// for (NULL: not).  Host pointers in the synchronous calls, device pointers in the sharded ones.
struct WhyOut { uint8_t* pair_why; uint32_t* pair_claim; uint32_t* pod_why; uint32_t* claim_blocks; };

// A reasons call (w; nullptr: the plain call, which answers no pair) with n_why pairs to answer needs pair_why
int why_check(dra_ctx* ctx, const WhyOut* w, uint32_t n_why) {
    if (w && n_why && !w->pair_why) return fail(ctx, DRA_E_INVAL, "pair_why is NULL");
    return DRA_OK;
}

// n_why: the pairs a place-pods call answers (spec §18; none without w): every pod at every node in the dense form
int place_why_pairs(dra_ctx* ctx, const WhyOut* w, bool dense, uint32_t n_pod, uint32_t n_pair, uint32_t& n_why) {
    const uint64_t n = !w ? 0 : dense ? (uint64_t)n_pod * ctx->n_node : n_pair;
    if (n > 0xFFFFFFFFull) return fail(ctx, DRA_E_INVAL, "%llu (pod, node) pairs: more than %llu", (unsigned long long)n, 0xFFFFFFFFull);
    n_why = (uint32_t)n;
    return DRA_OK;
}

// The device buffers of w's outputs (none without w) for n_why pairs, n_pod pods and n_claim claims, and their
// read-backs appended to outs: pair_why for every pair, each other output only when asked for
int why_buffers(dra_ctx* ctx, const WhyOut* w, Outputs& outs, uint32_t n_why, uint32_t n_pod, uint32_t n_claim) {
    if (!w) return DRA_OK;
    int rc;
    if ((rc = grow_set(ctx, ctx->cap_why_pairs, (size_t)n_why + 8, ctx->d_why, ctx->d_why_claim)) ||
        (rc = grow_set(ctx, ctx->cap_why_pods, (size_t)n_pod * DRA_WHY_N + 8, ctx->d_why_pod)) ||
        (rc = grow_set(ctx, ctx->cap_why_claims, (size_t)n_claim + 8, ctx->d_why_blocks))) return rc;
    outs.add(w->pair_why, ctx->d_why, n_why);
    outs.add(w->pair_claim, ctx->d_why_claim, w->pair_claim ? (size_t)n_why * 4 : 0);
    outs.add(w->pod_why, ctx->d_why_pod, w->pod_why ? (size_t)n_pod * DRA_WHY_N * 4 : 0);
    outs.add(w->claim_blocks, ctx->d_why_blocks, w->claim_blocks ? (size_t)n_claim * 4 : 0);
    return DRA_OK;
}

// The tallies of w, when pod_why or claim_blocks is asked for: d_why_blocks zeroed (in these calls only k_why_tally writes
// it, so just before it is soon enough), then k_why_tally over the records the walk wrote.  cand_off: the staged
// candidates' offsets, nullptr in the dense form.  Enqueues only.
int launch_why_tally(dra_ctx* ctx, const WhyOut& w, const uint32_t* cand_off, uint32_t n_pod, uint32_t n_claim) {
    if (!w.pod_why && !w.claim_blocks) return DRA_OK;
    if (w.claim_blocks && n_claim) CU(cudaMemsetAsync(ctx->d_why_blocks, 0, (size_t)n_claim * 4, ctx->stream));
    const WhyTally t{ctx->d_why, ctx->d_why_claim, cand_off, n_pod, ctx->n_node, w.pod_why ? ctx->d_why_pod : nullptr,
                     w.claim_blocks ? ctx->d_why_blocks : nullptr};
    k_why_tally<<<n_pod / 8 + 1, 256, 0, ctx->stream>>>(t);
    ctx->launches += 1;
    return DRA_OK;
}

// A sharded call at world > 1 needs the sharded form of the peer buffer, exported and imported
int need_peers(dra_ctx* ctx) {
    if (ctx->world <= 1 || (ctx->peer_ready && ctx->peer_form == 2)) return DRA_OK;
    return fail(ctx, DRA_E_STATE, "dra_shard_export + dra_peer_import have not been called");
}

// k_peer_push's grid for n units: a CTA per 256, at most two per SM
uint32_t push_grid(const dra_ctx* ctx, uint32_t n) { return std::max(1u, std::min((n + 255) / 256, (uint32_t)ctx->n_sm * 2u)); }

// The grid of a kernel that waits for its peers, for work CTAs' worth of work: at most SMs / 4 CTAs, because ranks
// sharing one device must not find the SMs of their own evaluation, walk, sort or push held by a peer's waiting CTAs
uint32_t wait_grid(const dra_ctx* ctx, size_t work) {
    return (uint32_t)std::max<size_t>(1, std::min<size_t>(work, (size_t)std::max(1, ctx->n_sm / 4)));
}

// A setter of the sizes dra_shard_export reserves: at world > 1, only before the export
int check_before_export(dra_ctx* ctx, const char* setter) {
    if (ctx->world > 1 && ctx->peer_local) return fail(ctx, DRA_E_STATE, "%s: call it before dra_shard_export", setter);
    return DRA_OK;
}

// The candidates of a sharded call, as device pointers: cand_nodes and cand_off both or neither (the dense form), at most
// 0xFFFFFFF0 pairs.  dense_all: the dense form has n_pair == n_pod * n_node pairs, else it gives n_pair 0.
int check_dev_cands(dra_ctx* ctx, const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t n_pod, uint32_t n_pair,
                    bool dense_all, bool& dense) {
    dense = cand_nodes == nullptr && cand_off == nullptr;
    if (!dense && (!cand_nodes || !cand_off)) return fail(ctx, DRA_E_INVAL, "cand_nodes and cand_off: both or neither");
    if (dense && dense_all && (uint64_t)n_pod * ctx->n_node != n_pair)
        return fail(ctx, DRA_E_INVAL, "dense form: n_pair %u != n_pod %u x n_node %u", n_pair, n_pod, ctx->n_node);
    if (dense && !dense_all && n_pair) return fail(ctx, DRA_E_INVAL, "dense form: n_pair must be 0");
    if (n_pair > 0xFFFFFFF0u) return fail(ctx, DRA_E_INVAL, "too many (pod, node) pairs");
    return DRA_OK;
}

// The inventory sync's exchange: reserved by dra_shard_export for the inventory loaded then, which has not grown since
int check_inv_exchange(dra_ctx* ctx) {
    if (!ctx->peer_inv_gpus) return fail(ctx, DRA_E_STATE, "the inventory was not loaded before dra_shard_export: the export reserved no staging for it");
    if (ctx->n_gpu > ctx->peer_inv_gpus)
        return fail(ctx, DRA_E_STATE, "the inventory grew to %u GPUs after dra_shard_export reserved staging for %u", ctx->n_gpu, ctx->peer_inv_gpus);
    return DRA_OK;
}

constexpr auto no_check = [] { return (int)DRA_OK; };

// What a sharded call needs at world > 1 besides its arguments, in this order: dra_set_shard_map (map_use: what needs every
// rank's range; nullptr: nothing does), a map spanning the inventory (spanning), the peers, reserved() (the call's
// exchange reserved by its setter before the export), n_out within the exported table (n_out < 0: the call has no table),
// fits() (the call within the reserved sizes).
template <class Reserved, class Fits>
int check_world(dra_ctx* ctx, const char* map_use, bool spanning, Reserved reserved, int64_t n_out, Fits fits) {
    if (ctx->world <= 1) return DRA_OK;
    if (map_use && !ctx->shard_map_on)
        return fail(ctx, DRA_E_STATE, "world > 1: dra_set_shard_map has not been called (%s every rank's range)", map_use);
    if (int rc = need_peers(ctx)) return rc;
    if (spanning && ctx->shard_bounds[ctx->world] != ctx->n_node)
        return fail(ctx, DRA_E_STATE, "the shard map does not span the inventory's %u nodes", ctx->n_node);
    if (int rc = reserved()) return rc;
    if (n_out > (int64_t)ctx->peer_tab_len) return fail(ctx, DRA_E_INVAL, "n_out %u exceeds the exported table (%u)", (uint32_t)n_out, ctx->peer_tab_len);
    return fits();
}

// The scope of a sharded call that enqueues: open() sets its device, and uploads the table.  Peers on this device may
// already wait for this rank (gather: world > 1), so no buffer the call outgrows is freed before the next dra_ctx_sync
// (defer_free, cleared when the scope ends).
struct CallScope {
    dra_ctx* ctx;
    ~CallScope() { ctx->defer_free = false; }
    int open(bool gather) {
        CU(cudaSetDevice(ctx->device));
        ctx->defer_free = gather;
        return upload_table(ctx);
    }
};

}  // namespace

namespace {
// Dynamic shared-memory limits are raised ONCE per device to the opt-in maximum, when a context is created: the attribute
// is per function, not per context — a lazily "grown" per-context value would LOWER it under another context's feet
template <class K>
int raise_one(dra_ctx* ctx, K k, int optin) {
    cudaFuncAttributes fa;
    CU(cudaFuncGetAttributes(&fa, k));
    const int dyn = optin - (int)fa.sharedSizeBytes;          // the opt-in limit covers static + dynamic
    if (dyn > 48 * 1024) CU(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
    return DRA_OK;
}
int raise_smem_limits(dra_ctx* ctx, int optin) {
    int rc;
    if ((rc = raise_one(ctx, k_fused<FUSED_NW, true>, optin))) return rc;
    if ((rc = raise_one(ctx, k_fused<FUSED_NW, false>, optin))) return rc;
    if ((rc = raise_one(ctx, k_bucket_small, optin))) return rc;
    if ((rc = raise_one(ctx, k_bucket_hist8<false>, optin))) return rc;
    if ((rc = raise_one(ctx, k_bucket_hist8<true>, optin))) return rc;
    if ((rc = raise_one(ctx, k_bucket_hist, optin))) return rc;
    if ((rc = raise_one(ctx, k_serve<FUSED_NW>, optin))) return rc;
    // The compaction runs right before the single-launch kernel, which wants the SM's L1/shared split at "all shared".  An SM
    // cannot hold CTAs of kernels with different splits at once: with the default split the dependent kernel's CTAs could
    // not be placed early (programmatic dependent launch) and the SMs were re-configured in between (profiles/tail_timeline.py
    // shows the gap from the compaction's last CTA to k_fused's first).  Same split for both.
    CU(cudaFuncSetAttribute(k_shard_compact_flat<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CU(cudaFuncSetAttribute(k_shard_compact_flat<8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CU(cudaFuncSetAttribute(k_shard_compact, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    return DRA_OK;
}

// ---- resident mode -----------------------------------------------------------------------------------------------
// Stops the resident kernel (if any): EXIT command, then wait for the kernel to leave.  Every entry point that launches
// other work or touches device state calls this first — the resident kernel owns the SMs' shared memory while it runs.
int serve_stop(dra_ctx* ctx) {
    if (!ctx->serve_on) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    if (ctx->h_stat[1] != 2u) {
        ServeCmd* c = ctx->h_cmd;
        c->n_claim = 0; c->n_out = 0; c->flags = SERVE_EXIT; c->claims = 0; c->out_off = 0; c->out = 0;
        __atomic_store_n(&c->seq, ctx->serve_seq + 1u, __ATOMIC_RELEASE);
    }
    CU(cudaStreamSynchronize(ctx->serve_stream));
    ctx->serve_on = false;
    ctx->serve_seq += 1;                        // the EXIT consumed a sequence number (or none was taken: harmless gap)
    return DRA_OK;
}

// largest claim count whose staged layout fits the single-launch kernel's shared memory
uint32_t serve_capacity() {
    uint32_t lo = 256, hi = FUSED_NW * FU_PIECE * FU_MAXPIECE;
    while (lo < hi) { const uint32_t mid = (lo + hi + 1) / 2; if (fused_smem_bytes(mid, FUSED_NW, true) <= 225 * 1024) lo = mid; else hi = mid - 1; }
    return lo;
}

int serve_start(dra_ctx* ctx) {
    CU(cudaSetDevice(ctx->device));
    if (!ctx->serve_stream) CU(cudaStreamCreateWithFlags(&ctx->serve_stream, cudaStreamNonBlocking));
    if (!ctx->h_cmd) {
        void* p = nullptr;
        CU(cudaHostAlloc(&p, 256, cudaHostAllocMapped));
        memset(p, 0, 256);
        ctx->h_cmd = (ServeCmd*)p; ctx->h_stat = (volatile uint32_t*)((uint8_t*)p + 128);
        void* dp = nullptr;
        CU(cudaHostGetDevicePointer(&dp, p, 0));
        ctx->h_cmd_dev = (ServeCmd*)dp; ctx->h_stat_dev = (uint32_t*)((uint8_t*)dp + 128);
        CU(cudaMalloc((void**)&ctx->d_go, 256)); CU(cudaMemset(ctx->d_go, 0, 256));
    }
    if (!ctx->d_gbar) { CU(cudaMalloc((void**)&ctx->d_gbar, 64)); CU(cudaMemset(ctx->d_gbar, 0, 64)); }
    int rc = upload_table(ctx);
    if (rc) return rc;
    CU(cudaStreamSynchronize(ctx->stream));                  // earlier work of this context is done before the kernel takes over
    ctx->serve_cap = serve_capacity();
    ctx->serve_smem = fused_smem_bytes(ctx->serve_cap, FUSED_NW, true);
    if ((rc = ensure_batch(ctx, ctx->serve_cap, ctx->serve_cap * 2, true))) return rc;
    ServeArgs sa; memset(&sa, 0, sizeof sa);
    PackArgs& a = sa.base;
    a.inv_dst = ctx->d_inv_live; a.inv_src = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.tbl = ctx->d_tbl;
    a.out = ctx->d_out; a.n_node = ctx->n_node; a.err = err_of(ctx); a.sel = sel_of(ctx);
    a.claims = ctx->d_claims;
    a.dio.d_claims = ctx->d_claims; a.dio.d_out_off = ctx->d_out_off; a.dio.gbar = ctx->d_gbar;
    sa.inv_pristine = ctx->d_inv_pristine;
    sa.h_cmd = ctx->h_cmd_dev; sa.h_stat = ctx->h_stat_dev; sa.d_go = ctx->d_go;
    sa.first_seq = ctx->serve_seq + 1; sa.cap_claims = ctx->serve_cap;
    static const long long idle_ms = getenv("DRA_SERVE_IDLE_MS") ? atoll(getenv("DRA_SERVE_IDLE_MS")) : 20;
    sa.idle_cycles = std::max(1ll, idle_ms) * 1900000ll;
    ctx->h_stat[1] = 0; ctx->h_stat[2] = 0;
    CU(cudaMemsetAsync(ctx->d_go, 0, 256, ctx->serve_stream));
    CU(launch_k(k_serve<FUSED_NW>, dim3(ctx->n_node + 1), dim3(FUSED_NW * 32), ctx->serve_smem, ctx->serve_stream, LA_COOP, sa));
    ctx->launches += 1;
    ctx->serve_on = true; ctx->serve_epoch = ctx->state_epoch;
    return DRA_OK;
}

// one batch through the resident kernel; *took = false when the kernel had gone idle before it saw the doorbell
int serve_call(dra_ctx* ctx, const void* src_c, uint32_t n_claim, const void* src_o, void* dst_o, uint32_t n_out, uint32_t flags) {
    for (int attempt = 0; attempt < 3; ++attempt) {
        if (!ctx->serve_on || ctx->h_stat[1] == 2u || ctx->serve_epoch != ctx->state_epoch) {
            int rc = serve_stop(ctx);
            if (rc) return rc;
            if ((rc = serve_start(ctx))) return rc;
        }
        const uint32_t seq = ctx->serve_seq + 1u;
        ServeCmd* c = ctx->h_cmd;
        c->n_claim = n_claim; c->n_out = n_out; c->flags = flags & DRA_F_FRESH_INVENTORY;
        c->claims = (unsigned long long)(uintptr_t)src_c; c->out_off = (unsigned long long)(uintptr_t)src_o; c->out = (unsigned long long)(uintptr_t)dst_o;
        __atomic_store_n(&c->seq, seq, __ATOMIC_RELEASE);                  // the doorbell
        uint64_t spins = 0;
        bool done = false, gone = false;
        while (true) {
            if (__atomic_load_n((const uint32_t*)&ctx->h_stat[0], __ATOMIC_ACQUIRE) == seq) { done = true; break; }
            if ((++spins & 0xFFu) == 0) {
                if (ctx->h_stat[1] == 2u) { gone = __atomic_load_n((const uint32_t*)&ctx->h_stat[0], __ATOMIC_ACQUIRE) != seq; if (gone) break; done = true; break; }
                if (spins > (1ull << 31)) return fail(ctx, DRA_E_CUDA, "resident kernel does not answer");
            }
        }
        if (done) { ctx->serve_seq = seq; ctx->serve_batches++; ctx->chain |= DRA_K_SERVE; return DRA_OK; }
        // the kernel left (idle time-out) before it saw this doorbell: start it again and ring once more
        CU(cudaStreamSynchronize(ctx->serve_stream));
        ctx->serve_on = false;
    }
    return fail(ctx, DRA_E_CUDA, "resident kernel keeps leaving before it takes the batch");
}

// Whether a kernel can read the caller's claims (src_c) and offsets (src_o, or NULL) and write its OutRecs (dst_o) in these
// host buffers as they are: 16-byte aligned records, 4-byte aligned offsets, and pointers the device can use unchanged
// (UVA identity mapping; checked once each)
bool host_io_ok(dra_ctx* ctx, const void* src_c, const void* src_o, void* dst_o) {
    if (((uintptr_t)src_c & 15) || ((uintptr_t)dst_o & 15) || ((uintptr_t)src_o & 3)) return false;
    const void* hp[3] = {src_c, src_o, dst_o};
    for (int k = 0; k < 3; ++k) {
        if (!hp[k] || ctx->dio_seen[k] == hp[k]) continue;
        void* dp = nullptr;
        if (cudaHostGetDevicePointer(&dp, const_cast<void*>(hp[k]), 0) != cudaSuccess || dp != hp[k]) { (void)cudaGetLastError(); return false; }
        ctx->dio_seen[k] = hp[k];
    }
    return true;
}

#define QUIESCE() do { int q_ = serve_stop(ctx); if (q_) return q_; } while (0)
}  // namespace

extern "C" {

int dra_abi_version(void) { return (int)DRA_ABI_VERSION; }

const char* dra_last_error(const dra_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int dra_ctx_create(const dra_cfg* cfg, dra_ctx** out) {
    dra_ctx* ctx = nullptr;   // for CU(): errors go to the thread-local create error
    if (!cfg || !out) return fail(nullptr, DRA_E_INVAL, "null argument");
    if (cfg->abi_version != DRA_ABI_VERSION) return fail(nullptr, DRA_E_INVAL, "abi_version %u != %u", cfg->abi_version, DRA_ABI_VERSION);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, DRA_E_CUDA, "no CUDA device (%s); this library has no CPU fallback", cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, DRA_E_INVAL, "device %d out of range", cfg->device);
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, DRA_E_CUDA, "device %d is sm_%d%d; this build is sm_90a only", cfg->device, prop.major, prop.minor);
    CU(cudaSetDevice(cfg->device));
    dra_ctx* c = new dra_ctx();
    c->device = cfg->device;
    c->cfg_flags = cfg->flags;
    c->n_sm = prop.multiProcessorCount;
    c->coop_ok = prop.cooperativeLaunch && prop.unifiedAddressing && prop.canUseHostPointerForRegisteredMem;
    ctx = c;
    auto bail = [&](int rc) { g_create_err = c->err; dra_ctx_destroy(c); return rc; };
    { int rc = raise_smem_limits(c, (int)prop.sharedMemPerBlockOptin); if (rc) return bail(rc); }
    if (cfg->stream) c->stream = (cudaStream_t)cfg->stream;
    else {
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(fail(c, DRA_E_CUDA, "cudaStreamCreate"));
        c->own_stream = true;
    }
    memset(c->h_tbl, 0, sizeof c->h_tbl);
    if (cudaMalloc((void**)&c->d_tbl, sizeof c->h_tbl) != cudaSuccess) return bail(fail(c, DRA_E_NOMEM, "cudaMalloc table"));
    if (cudaMalloc((void**)&c->d_err, ERR_WORDS * sizeof(uint32_t)) != cudaSuccess) return bail(fail(c, DRA_E_NOMEM, "cudaMalloc err"));
    cudaMemset(c->d_err, 0, ERR_WORDS * sizeof(uint32_t));
    void* he = nullptr;
    if (cudaHostAlloc(&he, ERR_WORDS * sizeof(uint32_t), cudaHostAllocMapped) != cudaSuccess) return bail(fail(c, DRA_E_NOMEM, "cudaHostAlloc err"));
    c->h_err = (volatile uint32_t*)he;
    for (uint32_t i = 0; i < ERR_WORDS; ++i) c->h_err[i] = 0;
    if (cudaHostGetDevicePointer((void**)&c->h_err_dev, he, 0) != cudaSuccess) return bail(fail(c, DRA_E_CUDA, "cudaHostGetDevicePointer"));
    if (cudaMalloc((void**)&c->d_ticket, 64) != cudaSuccess) return bail(fail(c, DRA_E_NOMEM, "cudaMalloc ticket"));
    cudaMemset(c->d_ticket, 0, 64);
    for (int i = 0; i < 8; ++i) if (cudaEventCreate(&c->ev[i]) != cudaSuccess) return bail(fail(c, DRA_E_CUDA, "cudaEventCreate"));
    c->ev_ok = true;
    if (cfg->max_claims) { int rc = ensure_batch(c, cfg->max_claims, cfg->max_claims, true); if (rc) return bail(rc); }
    *out = c;
    return DRA_OK;
}

void dra_ctx_destroy(dra_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    (void)serve_stop(c);
    if (c->serve_stream) cudaStreamDestroy(c->serve_stream);
    if (c->h_cmd) cudaFreeHost(c->h_cmd);
    if (c->d_go) cudaFree(c->d_go);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->graph_exec) cudaGraphExecDestroy(c->graph_exec);
    if (c->comm) { std::lock_guard<std::mutex> lk(g_nccl_mu); if (g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm); }
    for (int r = 0; r < (int)PEER_MAX; ++r) if (c->peer_base[r] && c->peer_ipc[r]) cudaIpcCloseMemHandle(c->peer_base[r]);
    if (c->peer_local) cudaFree(c->peer_local);
    if (c->d_ticket) cudaFree(c->d_ticket);
    if (c->d_scan_status) cudaFree(c->d_scan_status);
    if (c->d_gbar) cudaFree(c->d_gbar);
    void* dev[] = {c->d_inv_live, c->d_inv_pristine, c->d_node_off, c->d_tbl, c->d_claims, c->d_sorted, c->d_out_off,
                   c->d_out, c->d_rank, c->d_hist, c->d_claim_off, c->d_pod_off, c->d_cand_off, c->d_cand_nodes,
                   c->d_pair_pod, c->d_bits, c->d_err, c->d_attrs, c->d_sels, c->d_podrec, c->d_cursor, c->d_cclaims, c->d_coff,
                   c->d_sc_status, c->d_sc_counts, c->d_gtable, c->d_rank_slots, c->d_sc_times, c->d_ubits, c->d_upair_pod, c->d_spod,
                   c->d_place_state, c->d_place_node, c->d_place_cursor, c->d_splace_local, c->d_splace_rec,
                   c->d_pre_prio, c->d_pre_node, c->d_pre_nvic, c->d_pre_choice, c->d_pre_pst, c->d_pre_psum, c->d_pre_psum64,
                   c->d_pre_pairst, c->d_pre_pairvic, c->d_pre_rclaims, c->d_pre_routoff, c->d_pre_rpodoff, c->d_pre_rprio,
                   c->d_pre_rrec, c->d_pre_vlist, c->d_pre_rout, c->d_pre_vic, c->d_spre_part, c->d_pre_podviol,
                   c->d_pre_pairviol, c->d_pre_rpdb, c->d_pre_vprev, c->d_pre_allowed,
                   c->d_pp_pending, c->d_pp_evicted, c->d_pp_runoff, c->d_pp_judged, c->d_spp_inv, c->d_spp_gate,
                   c->d_cap_copies, c->d_cap_stop, c->d_cap_total, c->d_cap_nodes, c->d_scap_part,
                   c->d_why, c->d_why_claim, c->d_why_pod, c->d_why_blocks, c->d_swhy_part, c->d_swhy_blocks};
    for (void* p : dev) if (p) cudaFree(p);
    for (void* p : c->retired) cudaFree(p);
    if (c->h_err) cudaFreeHost((void*)c->h_err);
    if (c->h_sc_counts) cudaFreeHost((void*)c->h_sc_counts);
    if (c->h_in) cudaFreeHost(c->h_in);
    if (c->h_out) cudaFreeHost(c->h_out);
    if (c->ev_ok) for (int i = 0; i < 8; ++i) cudaEventDestroy(c->ev[i]);
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

int dra_set_placement_table(dra_ctx* ctx, uint32_t model, const dra_profile_tbl* tbl) {
    if (!ctx || !tbl) return DRA_E_INVAL;
    QUIESCE();
    if (model >= DRA_MAX_MODELS) return fail(ctx, DRA_E_INVAL, "model %u >= %u", model, DRA_MAX_MODELS);
    for (uint32_t p = 0; p < DRA_MAX_PROFILES; ++p) {
        const dra_prof_ent& e = tbl->ent[p];
        if (!e.start_mask) continue;
        if (e.size < 1 || e.size > 16) return fail(ctx, DRA_E_INVAL, "profile %u: size %u", p, e.size);
        int hi = 15; while (!((e.start_mask >> hi) & 1)) --hi;
        if (hi + e.size > 16) return fail(ctx, DRA_E_INVAL, "profile %u: start %d + size %u > 16", p, hi, e.size);
    }
    ctx->h_tbl[model] = *tbl;
    ctx->tbl_dirty = true;
    ctx->state_epoch++;
    return DRA_OK;
}

int dra_set_inventory(dra_ctx* ctx, const dra_gpu_rec* gpus, uint32_t n_gpu, const uint32_t* node_off, uint32_t n_node) {
    if (!ctx || !node_off || (n_gpu && !gpus)) return DRA_E_INVAL;
    QUIESCE();
    CU(cudaSetDevice(ctx->device));
    if (node_off[0] != 0 || node_off[n_node] != n_gpu) return fail(ctx, DRA_E_INVAL, "node_off must span [0, n_gpu]");
    for (uint32_t n = 0; n < n_node; ++n) {
        if (node_off[n + 1] < node_off[n]) return fail(ctx, DRA_E_INVAL, "node_off not monotone at node %u", n);
        if (node_off[n + 1] - node_off[n] > DRA_MAX_GPUS_PER_NODE) return fail(ctx, DRA_E_INVAL, "node %u has more than %u GPUs", n, DRA_MAX_GPUS_PER_NODE);
        for (uint32_t g = node_off[n]; g < node_off[n + 1]; ++g) {
            if (gpus[g].model >= DRA_MAX_MODELS) return fail(ctx, DRA_E_INVAL, "gpu %u: model %u", g, gpus[g].model);
            if (gpus[g].node != n) return fail(ctx, DRA_E_INVAL, "gpu %u: node field %u, expected %u", g, gpus[g].node, n);
        }
    }
    CU(cudaStreamSynchronize(ctx->stream));
    if (n_gpu + 8 > ctx->cap_nodes || !ctx->d_inv_live) {   // cap_nodes doubles as "inventory capacity"
        if (ctx->d_inv_live) CU(cudaFree(ctx->d_inv_live));
        if (ctx->d_inv_pristine) CU(cudaFree(ctx->d_inv_pristine));
        ctx->d_inv_live = ctx->d_inv_pristine = nullptr;
        size_t cap = (size_t)n_gpu + 64;
        CU(cudaMalloc((void**)&ctx->d_inv_live, cap * 16));
        CU(cudaMalloc((void**)&ctx->d_inv_pristine, cap * 16));
        ctx->cap_nodes = cap;
    }
    if (ctx->d_node_off) CU(cudaFree(ctx->d_node_off));
    if (ctx->d_claim_off) CU(cudaFree(ctx->d_claim_off));
    ctx->d_node_off = ctx->d_claim_off = nullptr;
    CU(cudaMalloc((void**)&ctx->d_node_off, ((size_t)n_node + 8) * 4));
    CU(cudaMalloc((void**)&ctx->d_claim_off, ((size_t)n_node + 8) * 4));
    if (n_gpu) CU(cudaMemcpy(ctx->d_inv_pristine, gpus, (size_t)n_gpu * 16, cudaMemcpyHostToDevice));
    if (n_gpu) CU(cudaMemcpy(ctx->d_inv_live, gpus, (size_t)n_gpu * 16, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(ctx->d_node_off, node_off, ((size_t)n_node + 1) * 4, cudaMemcpyHostToDevice));
    ctx->h_node_off.assign(node_off, node_off + n_node + 1);
    ctx->n_gpu = n_gpu; ctx->n_node = n_node;
    ctx->state_epoch++;
    ctx->max_width = 0;
    for (uint32_t n = 0; n < n_node; ++n) ctx->max_width = std::max(ctx->max_width, node_off[n + 1] - node_off[n]);
    ctx->cap_hist = 0;  // histogram geometry depends on n_node
    if (ctx->d_hist) { CU(cudaFree(ctx->d_hist)); ctx->d_hist = nullptr; }
    return DRA_OK;
}

int dra_set_gpu_attrs(dra_ctx* ctx, const dra_gpu_attr* attrs, uint32_t n_gpu) {
    if (!ctx || (n_gpu && !attrs)) return DRA_E_INVAL;
    QUIESCE();
    static_assert(sizeof(dra_gpu_attr) == 16 && sizeof(dra_selector) == 64, "selector record layout");
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->d_attrs) { CU(cudaFree(ctx->d_attrs)); ctx->d_attrs = nullptr; }
    ctx->n_attr = 0;
    ctx->state_epoch++;                      // a captured graph holds the freed pointer: never replay it
    if (!n_gpu) return DRA_OK;
    CU(cudaMalloc((void**)&ctx->d_attrs, (size_t)n_gpu * 16 + 64));
    CU(cudaMemcpy(ctx->d_attrs, attrs, (size_t)n_gpu * 16, cudaMemcpyHostToDevice));
    ctx->n_attr = n_gpu;
    ctx->state_epoch++;
    return DRA_OK;
}

int dra_set_selectors(dra_ctx* ctx, const dra_selector* sels, uint32_t n_sel) {
    if (!ctx || (n_sel && !sels)) return DRA_E_INVAL;
    QUIESCE();
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->d_sels) { CU(cudaFree(ctx->d_sels)); ctx->d_sels = nullptr; }
    ctx->n_sel = 0;
    ctx->state_epoch++;
    if (!n_sel) return DRA_OK;
    CU(cudaMalloc((void**)&ctx->d_sels, (size_t)n_sel * 64 + 64));
    CU(cudaMemcpy(ctx->d_sels, sels, (size_t)n_sel * 64, cudaMemcpyHostToDevice));
    ctx->n_sel = n_sel;
    ctx->state_epoch++;
    return DRA_OK;
}

int dra_get_inventory(dra_ctx* ctx, dra_gpu_rec* gpus, uint32_t n_gpu) {
    if (!ctx || !gpus) return DRA_E_INVAL;
    QUIESCE();
    if (n_gpu != ctx->n_gpu) return fail(ctx, DRA_E_INVAL, "n_gpu %u != inventory size %u", n_gpu, ctx->n_gpu);
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (n_gpu) CU(cudaMemcpy(gpus, ctx->d_inv_live, (size_t)n_gpu * 16, cudaMemcpyDeviceToHost));
    return DRA_OK;
}

int dra_reset_inventory(dra_ctx* ctx) {
    if (!ctx) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "no inventory");
    CU(cudaSetDevice(ctx->device));
    if (ctx->n_gpu) CU(cudaMemcpyAsync(ctx->d_inv_live, ctx->d_inv_pristine, (size_t)ctx->n_gpu * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    return DRA_OK;
}

int dra_ctx_sync(dra_ctx* ctx) {
    if (!ctx) return DRA_E_INVAL;
    QUIESCE();
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    std::vector<void*> retired; retired.swap(ctx->retired);
    for (void* p : retired) CU(cudaFree(p));
    collect_timings(ctx, 5);
    return check_err(ctx);
}

int dra_allocate_batch_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim, const uint32_t* d_out_off,
                              dra_out_rec* d_out, uint32_t n_out, uint32_t flags) {
    if (!ctx || (n_claim && (!d_claims || !d_out))) return DRA_E_INVAL;
    QUIESCE();
    ctx->chain = ctx->chain_tile = 0;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_batch(ctx, n_claim, n_out, false);
    if (rc) return rc;
    return launch_allocate(ctx, (const uint4*)d_claims, n_claim, d_out_off, (uint2*)d_out, n_out, flags);
}

int dra_allocate_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* out_off,
                       dra_out_rec* out, uint32_t n_out, uint32_t flags) {
    if (!ctx || (n_claim && (!claims || !out))) return DRA_E_INVAL;
    if (!out_off && n_out < n_claim) return fail(ctx, DRA_E_INVAL, "n_out %u < n_claim %u without out_off", n_out, n_claim);
    ctx->chain = ctx->chain_tile = 0;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_batch(ctx, n_claim, n_out, true);
    if (rc) return rc;
    const size_t cb = (size_t)n_claim * 16, ob = out_off ? (size_t)n_claim * 4 : 0, rb = (size_t)n_out * 8;
    // host -> device (staged through pinned memory unless the caller's buffers are dra_host_alloc'ed)
    const void* src_c = claims; const void* src_o = out_off;
    if (cb && !is_pinned(claims, cb)) {
        if ((rc = grow_pinned(ctx, ctx->h_in, ctx->h_in_cap, cb + ob))) return rc;
        memcpy(ctx->h_in, claims, cb); src_c = ctx->h_in;
        if (ob) { memcpy(ctx->h_in + cb, out_off, ob); src_o = ctx->h_in + cb; }
    } else if (ob && !is_pinned(out_off, ob)) {
        if ((rc = grow_pinned(ctx, ctx->h_in, ctx->h_in_cap, ob))) return rc;
        memcpy(ctx->h_in, out_off, ob); src_o = ctx->h_in;
    }
    const bool direct = rb && is_pinned(out, rb);
    if (rb && !direct && (rc = grow_pinned(ctx, ctx->h_out, ctx->h_out_cap, rb))) return rc;
    void* dst_o = direct ? (void*)out : (void*)ctx->h_out;

    // Resident mode (DRA_CFG_RESIDENT): the kernel is already up — write the command, ring the doorbell, spin on the
    // completion word.  Same eligibility as direct host I/O below; anything else stops the resident kernel first.
    {
        bool ok = (ctx->cfg_flags & DRA_CFG_RESIDENT) && ctx->coop_ok && n_claim && rb && !ctx->profiling && !getenv("DRA_TIMELINE") &&
                  !(flags & ~DRA_F_FRESH_INVENTORY) && (int)(ctx->n_node + 1) <= ctx->n_sm && ctx->d_inv_live;
        if (ok) {
            if (!ctx->serve_cap) ctx->serve_cap = serve_capacity();
            ok = n_claim <= ctx->serve_cap && n_out <= 2 * ctx->serve_cap && host_io_ok(ctx, src_c, src_o, dst_o);
        }
        if (ok) {
            rc = serve_call(ctx, src_c, n_claim, src_o, dst_o, n_out, flags);
            if (rc) return rc;
            if ((rc = check_err(ctx))) return rc;
            if (rb && !direct) memcpy(out, ctx->h_out, rb);
            return DRA_OK;
        }
        QUIESCE();
    }
    // Direct host I/O: when the batch takes the single-launch kernel with the claim array staged in shared memory
    // and all its CTAs can be resident at once, the kernel itself reads the claims from the (pinned, device-mapped)
    // host buffer and writes the OutRecs back there — no copy-engine transfers, no graph, one cooperative launch.
    {
        const FusedPlan plan = fused_plan(ctx, n_claim, flags, ctx->n_node);
        bool ok = !(ctx->cfg_flags & DRA_CFG_NO_DIRECT) && ctx->coop_ok && plan.fused && plan.stage && n_claim && rb && !ctx->profiling;
        int ctas = 0;
        if (ok && (rc = fused_resident_ctas(ctx, true, plan.smem, ctas))) return rc;
        ok = ok && (int)(ctx->n_node + 1) <= ctas && host_io_ok(ctx, src_c, src_o, dst_o);
        if (ok && !ctx->d_gbar) { CU(cudaMalloc((void**)&ctx->d_gbar, 64)); CU(cudaMemsetAsync(ctx->d_gbar, 0, 64, ctx->stream)); }
        if (ok) {
            DirectIO d;
            d.h_claims = (const uint4*)src_c; d.h_out_off = (const uint32_t*)src_o; d.h_out = (uint2*)dst_o;
            d.d_claims = ctx->d_claims; d.d_out_off = ctx->d_out_off; d.gbar = ctx->d_gbar;
            ctx->dio_pending = d;
            rc = launch_allocate(ctx, ctx->d_claims, n_claim, out_off ? ctx->d_out_off : nullptr, ctx->d_out, n_out, flags);
            ctx->dio_pending = DirectIO{};
            if (rc) return rc;
            CU(cudaStreamSynchronize(ctx->stream));
            if ((rc = check_err(ctx))) return rc;
            if (rb && !direct) memcpy(out, ctx->h_out, rb);
            return DRA_OK;
        }
    }

    // DRA_CFG_USE_GRAPH: H2D -> kernel chain -> D2H replayed as ONE cudaGraphLaunch when the call has the same
    // shape and buffers as the previous one (the first call of a shape runs eagerly: it also sets the kernels'
    // shared-memory attributes, which cannot happen inside a capture).
    GraphKey key{src_c, src_o, dst_o, n_claim, n_out, flags, ctx->state_epoch};
    const bool want_graph = (ctx->cfg_flags & DRA_CFG_USE_GRAPH) && !ctx->profiling && !getenv("DRA_TIMELINE");
    if (want_graph && ctx->graph_exec && key == ctx->graph_key) {
        CU(cudaGraphLaunch(ctx->graph_exec, ctx->stream));
        ctx->launches += ctx->graph_launches;
        ctx->chain = ctx->graph_chain; ctx->chain_tile = ctx->graph_tile;
    } else {
        const bool capture = want_graph && key == ctx->graph_key;      // second call of this shape: capture it
        if (want_graph && !capture) { ctx->graph_key = key; if (ctx->graph_exec) { cudaGraphExecDestroy(ctx->graph_exec); ctx->graph_exec = nullptr; } }
        const uint64_t l0 = ctx->launches;
        if (capture) CU(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
        cudaError_t ce = cudaSuccess;
        if (cb) ce = cudaMemcpyAsync(ctx->d_claims, src_c, cb, cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess && ob) ce = cudaMemcpyAsync(ctx->d_out_off, src_o, ob, cudaMemcpyHostToDevice, ctx->stream);
        if (ce == cudaSuccess) rc = launch_allocate(ctx, ctx->d_claims, n_claim, out_off ? ctx->d_out_off : nullptr, ctx->d_out, n_out, flags);
        if (ce == cudaSuccess && rc == DRA_OK && rb) ce = cudaMemcpyAsync(dst_o, ctx->d_out, rb, cudaMemcpyDeviceToHost, ctx->stream);
        if (capture) {
            cudaGraph_t g = nullptr;
            cudaError_t ee = cudaStreamEndCapture(ctx->stream, &g);
            if (ce != cudaSuccess || rc != DRA_OK || ee != cudaSuccess || !g) {
                if (g) cudaGraphDestroy(g);
                (void)cudaGetLastError();
                ctx->graph_key = GraphKey{};
                return rc != DRA_OK ? rc : fail(ctx, DRA_E_CUDA, "graph capture failed: %s", cudaGetErrorString(ce != cudaSuccess ? ce : ee));
            }
            ctx->graph_launches = (uint32_t)(ctx->launches - l0);
            ctx->graph_chain = ctx->chain; ctx->graph_tile = ctx->chain_tile;
            cudaError_t ie = cudaGraphInstantiate(&ctx->graph_exec, g, 0);
            cudaGraphDestroy(g);
            if (ie != cudaSuccess) { ctx->graph_exec = nullptr; return fail(ctx, DRA_E_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ie)); }
            CU(cudaGraphLaunch(ctx->graph_exec, ctx->stream));
        } else {
            if (ce != cudaSuccess) return fail(ctx, DRA_E_CUDA, "enqueue: %s", cudaGetErrorString(ce));
            if (rc) return rc;
        }
    }
    CU(cudaStreamSynchronize(ctx->stream));
    collect_timings(ctx, 4);
    if ((rc = check_err(ctx))) return rc;
    if (rb && !direct) memcpy(out, ctx->h_out, rb);
    return DRA_OK;
}

int dra_unsuitable_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, uint32_t n_pod,
                         const uint32_t* cand_nodes, const uint32_t* cand_off, uint8_t* suitable_bits, uint32_t flags) {
    if (!ctx || !pod_off || (n_claim && !claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_unsuitable_batch: unknown flags 0x%x", flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    bool dense; uint32_t n_pair;
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_cands(ctx, n_pod, cand_nodes, cand_off, 0xFFFFFFFFu, ctx->n_node, 0xFFFFFFF0ull, dense, n_pair))) return rc;
    if (n_pair && !suitable_bits) return fail(ctx, DRA_E_INVAL, "suitable_bits is NULL");
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, n_claim, 1, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    const size_t words = ((size_t)n_pair + 31) / 32;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (!dense && (rc = grow_set(ctx, ctx->cap_pairs, (size_t)n_pair + 64, ctx->d_cand_nodes, ctx->d_pair_pod))) ||
        (rc = grow_set(ctx, ctx->cap_bits_only, words + 8, ctx->d_bits))) return rc;
    Staging s;                                            // (cand_off is only needed on the host)
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    if (!dense) {
        s.add(ctx->d_cand_nodes, cand_nodes, (size_t)n_pair * 4);
        s.add(ctx->d_pair_pod, nullptr, (size_t)n_pair * 4);
    }
    if ((rc = stage_in(ctx, s, [&](uint8_t* h) { expand_pairs((uint32_t*)h, cand_off, n_pod); }))) return rc;
    if (n_pair) {
        CU(cudaMemsetAsync(ctx->d_bits, 0, words * 4, ctx->stream));
        UnsArgs a; memset(&a, 0, sizeof a);
        a.claims = ctx->d_claims; a.pod_off = ctx->d_pod_off; a.n_pod = n_pod;
        a.cand_nodes = ctx->d_cand_nodes; a.pair_pod = ctx->d_pair_pod;
        a.cand_off = dense ? nullptr : ctx->d_cand_off;   // (not staged: k_unsuitable reads only whether it is nullptr)
        a.inv = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.tbl = ctx->d_tbl; a.bits = ctx->d_bits;
        a.sel = sel_of(ctx);
        a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u;
        a.n_walk = n_pair;                                 // (the window is the whole inventory)
        Prof prof(ctx);
        if ((rc = launch_unsuitable(ctx, a, false))) return rc;
        prof.mark();
        if ((rc = grow_pinned(ctx, ctx->h_out, ctx->h_out_cap, words * 4))) return rc;
        CU(cudaMemcpyAsync(ctx->h_out, ctx->d_bits, words * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    // k_unsuitable sets no fault word (one left by an earlier enqueue-only call is dra_ctx_sync's to report)
    CU(cudaStreamSynchronize(ctx->stream));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "k_unsuitable: %s", cudaGetErrorString(e));
    collect_timings(ctx, 1);
    if (n_pair) memcpy(suitable_bits, ctx->h_out, ((size_t)n_pair + 7) / 8);
    return DRA_OK;
}

// Why each node is unsuitable (spec §17): every argument is checked here, before anything is staged or launched, so a
// rejected call writes nothing.  k_unsuitable's reasons instantiation writes a record per pair, k_why_tally the sums; the
// outputs reach the caller after one synchronise.
int dra_unsuitable_why_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, uint32_t n_pod,
                             const uint32_t* cand_nodes, const uint32_t* cand_off, uint8_t* pair_why, uint32_t* pair_claim,
                             uint32_t* pod_why, uint32_t* claim_blocks, uint32_t flags) {
    if (!ctx || !pod_off || (n_claim && !claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_unsuitable_why_batch: unknown flags 0x%x", flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    bool dense; uint32_t n_pair;
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_cands(ctx, n_pod, cand_nodes, cand_off, 0xFFFFFFFFu, ctx->n_node, 0xFFFFFFFFull, dense, n_pair))) return rc;
    const WhyOut w{pair_why, pair_claim, pod_why, claim_blocks};
    if ((rc = why_check(ctx, &w, n_pair))) return rc;
    ctx->chain = DRA_K_UNSUITABLE_WHY; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, n_claim, 1, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    Outputs outs;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (!dense && (rc = grow_set(ctx, ctx->cap_pairs, (size_t)n_pair + 64, ctx->d_cand_nodes, ctx->d_pair_pod))) ||
        (rc = why_buffers(ctx, &w, outs, n_pair, n_pod, n_claim)) ||
        (rc = reserve_out(ctx, outs))) return rc;
    Staging s;
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    if (!dense) {
        s.add(ctx->d_cand_off, cand_off, ((size_t)n_pod + 1) * 4);
        s.add(ctx->d_cand_nodes, cand_nodes, (size_t)n_pair * 4);
        s.add(ctx->d_pair_pod, nullptr, (size_t)n_pair * 4);
    }
    if ((rc = stage_in(ctx, s, [&](uint8_t* h) { expand_pairs((uint32_t*)h, cand_off, n_pod); }))) return rc;
    Prof prof(ctx);
    if (n_pair) {
        UnsArgs a; memset(&a, 0, sizeof a);
        a.claims = ctx->d_claims; a.pod_off = ctx->d_pod_off; a.n_pod = n_pod;
        a.cand_nodes = ctx->d_cand_nodes; a.pair_pod = ctx->d_pair_pod;
        a.cand_off = dense ? nullptr : ctx->d_cand_off;
        a.inv = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.tbl = ctx->d_tbl;
        a.sel = sel_of(ctx);
        a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u;
        a.n_walk = n_pair;                                 // (the window is the whole inventory)
        a.why = ctx->d_why; a.why_claim = ctx->d_why_claim;
        if ((rc = launch_unsuitable(ctx, a, false, true))) return rc;
    }
    if ((rc = launch_why_tally(ctx, w, dense ? nullptr : ctx->d_cand_off, n_pod, n_claim))) return rc;
    prof.mark();
    return read_back(ctx, "unsuitable reasons kernels", 1, outs);
}

// Allocate with pod boundaries (spec §12): pod records -> stable counting sort of the PODS by node (the claim path's
// bucketing kernels, the record has a ClaimRec's layout) -> one warp per node walks its pods in input order.  The slot
// ranges are checked here, before anything is enqueued (k_pod_records checks them again): k_pods does not look at the
// fault word, so a bad range found only on the device would leave every other pod applied and no OutRec returned.
int dra_allocate_pods_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, uint32_t n_pod,
                            const uint32_t* out_off, dra_out_rec* out, uint32_t n_out, uint32_t flags) {
    if (!ctx || !pod_off || (n_claim && (!claims || !out))) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~(DRA_F_EXHAUSTIVE | DRA_F_FRESH_INVENTORY)) return fail(ctx, DRA_E_INVAL, "dra_allocate_pods_batch: unknown flags 0x%x", flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_slots(ctx, claims, n_claim, out_off, n_out, false)) ||
        (rc = check_sortable(ctx, n_pod))) return rc;
    ctx->chain = ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, std::max(n_claim, n_pod), n_out, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (rc = grow_set(ctx, ctx->cap_podrec, (size_t)n_pod + 8, ctx->d_podrec))) return rc;
    const Outputs outs = {{out, ctx->d_out, (size_t)n_out * 8}};
    if ((rc = reserve_out(ctx, outs))) return rc;
    Staging s;
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    if (out_off) s.add(ctx->d_out_off, out_off, (size_t)n_claim * 4);
    if ((rc = stage_in(ctx, s))) return rc;
    const uint32_t owned_lo = out_off ? 0u : n_claim;    // slots no claim owns read back as 0 (without out_off: past n_claim)
    if (n_out > owned_lo) CU(cudaMemsetAsync(ctx->d_out + owned_lo, 0, (size_t)(n_out - owned_lo) * 8, ctx->stream));
    Err err = err_of(ctx);
    Prof prof(ctx);
    uint2* d_out = ctx->d_out;
    const uint32_t* d_oo = out_off ? ctx->d_out_off : nullptr;
    k_pod_records<<<(n_pod + 255) / 256, 256, 0, ctx->stream>>>(ctx->d_claims, ctx->d_pod_off, n_pod, ctx->n_node, d_oo, d_out, n_out, ctx->d_podrec, err);
    ctx->launches += 1;
    const uint4* inv_src = (flags & DRA_F_FRESH_INVENTORY) ? ctx->d_inv_pristine : ctx->d_inv_live;
    if ((rc = launch_sort(ctx, ctx->d_podrec, n_pod, nullptr, nullptr, 0, 0, prof, inv_src, LA_NONE, ctx->n_node, ctx->d_node_off))) return rc;
    PodArgs a; memset(&a, 0, sizeof a);
    a.claims = ctx->d_claims; a.out_off = d_oo; a.out = d_out;
    a.sorted = ctx->d_sorted; a.claim_off = ctx->d_claim_off;
    a.inv_src = inv_src; a.inv_dst = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.tbl = ctx->d_tbl;
    a.n_node = ctx->n_node; a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u; a.sel = sel_of(ctx); a.err = err;
    if (ctx->n_node) {
        const uint32_t grid = std::max(1u, std::min((ctx->n_node + 3) / 4, (uint32_t)ctx->n_sm * 8u));
        CU(launch_k(k_pods<4>, dim3(grid), dim3(128), 0, ctx->stream, pdl_attr(ctx), a));
        ctx->launches += 1;
    }
    prof.mark();                                          // the walk: the pack stage of the timings
    return read_back(ctx, "pod kernels", 4, outs);
}

// Place pods (spec §13): pod records -> (candidate form) the pair records stably sorted by node with the claim path's
// bucketing kernels -> one persistent cooperative launch in which each warp walks its nodes' visit lists.  Everything is
// validated here, before anything is enqueued: a rejected call changes nothing.  With why (spec §18) the walk is the
// reasons instantiation, which also answers every pair (the prep the pairs no walk reaches), k_why_tally sums them, and
// every output comes back after the same one synchronise.
namespace {
int place_pods_call(dra_ctx* ctx, const char* name, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off,
                    uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off, const uint32_t* out_off,
                    dra_out_rec* out, uint32_t n_out, uint32_t* pod_node, const WhyOut* why, uint32_t flags) {
    if (!ctx || !pod_off || (n_claim && (!claims || !out)) || (n_pod && !pod_node)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~(DRA_F_EXHAUSTIVE | DRA_F_FRESH_INVENTORY)) return fail(ctx, DRA_E_INVAL, "%s: unknown flags 0x%x", name, flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    bool dense; uint32_t n_pair;                          // the dense form walks every node, ascending: no pair records
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_cands(ctx, n_pod, cand_nodes, cand_off, PL_POS, 0, 0xFFFFFFF0ull, dense, n_pair))) return rc;
    if (ctx->n_node > PL_POS) return fail(ctx, DRA_E_INVAL, "more than %u nodes", PL_POS);
    if ((rc = check_slots(ctx, claims, n_claim, out_off, n_out, true)) ||
        (rc = check_sortable(ctx, dense ? 0 : n_pair))) return rc;
    uint32_t n_why;
    if ((rc = place_why_pairs(ctx, why, dense, n_pod, n_pair, n_why)) || (rc = why_check(ctx, why, n_why))) return rc;
    ctx->chain = ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;
    if (!ctx->coop_ok) return fail(ctx, DRA_E_STATE, "%s needs cooperative launches, which this device does not offer", name);
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, std::max(std::max(n_claim, n_pod), n_pair), n_out, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (rc = grow_set(ctx, ctx->cap_pairs, (size_t)n_pair + 64, ctx->d_cand_nodes, ctx->d_pair_pod)) ||
        (rc = grow_set(ctx, ctx->cap_podrec, (size_t)n_pair + 8, ctx->d_podrec)) ||
        (rc = grow_set(ctx, ctx->cap_place_pods, (size_t)n_pod + 8, ctx->d_place_state, ctx->d_place_node)) ||
        (rc = grow_set(ctx, ctx->cap_place_cursor, (size_t)ctx->n_node + 8, ctx->d_place_cursor))) return rc;
    const size_t rb = (size_t)n_out * 8;
    Outputs outs = {{out, ctx->d_out, rb}, {pod_node, ctx->d_place_node, (size_t)n_pod * 4}};
    if ((rc = why_buffers(ctx, why, outs, n_why, n_pod, n_claim)) || (rc = reserve_out(ctx, outs))) return rc;
    Staging s;
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    if (out_off) s.add(ctx->d_out_off, out_off, (size_t)n_claim * 4);
    if (!dense) {
        s.add(ctx->d_cand_off, cand_off, ((size_t)n_pod + 1) * 4);
        s.add(ctx->d_cand_nodes, cand_nodes, (size_t)n_pair * 4);
    }
    if ((rc = stage_in(ctx, s))) return rc;
    if (rb) CU(cudaMemsetAsync(ctx->d_out, 0, rb, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_place_cursor, 0, ((size_t)ctx->n_node + 1) * 4, ctx->stream));
    Prof prof(ctx);
    PlaceArgs a; memset(&a, 0, sizeof a);
    a.claims = ctx->d_claims; a.pod_off = ctx->d_pod_off; a.n_pod = n_pod;
    a.cand_nodes = dense ? nullptr : ctx->d_cand_nodes; a.cand_off = dense ? nullptr : ctx->d_cand_off;
    a.out_off = out_off ? ctx->d_out_off : nullptr; a.out = ctx->d_out;
    a.state = ctx->d_place_state; a.pod_node = ctx->d_place_node; a.pairs = ctx->d_podrec;
    a.sorted = ctx->d_sorted; a.list_off = ctx->d_claim_off; a.cursor = ctx->d_place_cursor;
    a.inv_src = (flags & DRA_F_FRESH_INVENTORY) ? ctx->d_inv_pristine : ctx->d_inv_live; a.inv_dst = ctx->d_inv_live;
    a.node_off = ctx->d_node_off; a.tbl = ctx->d_tbl;
    a.n_node = ctx->n_node; a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u; a.sel = sel_of(ctx); a.err = err_of(ctx);
    if (why) { a.why = ctx->d_why; a.why_claim = ctx->d_why_claim; }
    k_pods_place_prep<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, ctx->stream>>>(a);
    ctx->launches += 1;
    // A candidate form with no pair sorts nothing, so the visit lists are zeroed instead: the walk must not read the
    // offsets an earlier call's sort left in d_claim_off (an Allocate's claims by node), as lists of this call's pairs
    if (!dense && !n_pair) CU(cudaMemsetAsync(ctx->d_claim_off, 0, ((size_t)ctx->n_node + 2) * 4, ctx->stream));
    if (!dense && n_pair &&
        (rc = launch_sort(ctx, ctx->d_podrec, n_pair, nullptr, nullptr, 0, 0, prof, a.inv_src, LA_NONE, ctx->n_node, ctx->d_node_off)))
        return rc;
    if (!why) {
        if ((rc = launch_walk(ctx, ctx->place_occ, "k_pods_place", k_pods_place<4>, a, PlaceShard{}))) return rc;
        ctx->chain |= DRA_K_PLACE;
    } else {
        // (sized by its own occupancy: its registers are not k_pods_place<4>'s)
        if ((rc = launch_walk(ctx, ctx->place_why_occ, "k_pods_place<4, false, true>", k_pods_place<4, false, true>, a, PlaceShard{})) ||
            (rc = launch_why_tally(ctx, *why, dense ? nullptr : ctx->d_cand_off, n_pod, n_claim)))
            return rc;
        ctx->chain |= DRA_K_PLACE | DRA_K_PLACE_WHY;
    }
    prof.mark();
    return read_back(ctx, why ? "place reasons kernels" : "place kernels", 4, outs);
}
}  // namespace

int dra_place_pods_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, uint32_t n_pod,
                         const uint32_t* cand_nodes, const uint32_t* cand_off, const uint32_t* out_off, dra_out_rec* out,
                         uint32_t n_out, uint32_t* pod_node, uint32_t flags) {
    return place_pods_call(ctx, "dra_place_pods_batch", claims, n_claim, pod_off, n_pod, cand_nodes, cand_off, out_off, out, n_out,
                           pod_node, nullptr, flags);
}

// Why place pods put each pod where it did (spec §18): dra_place_pods_batch's call, every pair answered on the state its
// pod met
int dra_place_pods_why_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, uint32_t n_pod,
                             const uint32_t* cand_nodes, const uint32_t* cand_off, const uint32_t* out_off, dra_out_rec* out,
                             uint32_t n_out, uint32_t* pod_node, uint8_t* pair_why, uint32_t* pair_claim, uint32_t* pod_why,
                             uint32_t* claim_blocks, uint32_t flags) {
    const WhyOut w{pair_why, pair_claim, pod_why, claim_blocks};
    return place_pods_call(ctx, "dra_place_pods_why_batch", claims, n_claim, pod_off, n_pod, cand_nodes, cand_off, out_off, out,
                           n_out, pod_node, &w, flags);
}

// Preemption (spec §14): the pending-pod arrays are checked here; the running pods on the device (k_pre_running), whose
// fault gates every later kernel.  Inputs are staged in, the kernels launched, the outputs copied back after ONE
// synchronise, and the caller's buffers are written only when no fault was found.  With why (spec §19,
// dra_preempt_why_batch) the pairs are the reasons instantiation of k_pods_preempt, which stops at each pair's status;
// nothing is chosen and no victim row is built, and k_why_tally sums the records.
namespace {
int preempt_call(dra_ctx* ctx, const char* name, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off,
                 const int32_t* prio, uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off,
                 const dra_running_pods* running, const dra_disruption_budgets* budgets, uint8_t* pair_status,
                 uint32_t* pair_victims, uint32_t* pair_violations, uint32_t* pod_node, uint8_t* pod_status, uint32_t* n_victims,
                 uint32_t* pod_violations, uint32_t* victims, uint32_t max_victims, const WhyOut* why, uint32_t flags) {
    if (!ctx || !pod_off || !running || !running->pod_off || (n_claim && !claims) ||
        (n_pod && (!prio || (!why && (!pod_node || !pod_status || !n_victims)))))
        return DRA_E_INVAL;
    const dra_running_pods& R = *running;
    if ((R.n_claim && !R.claims) || (R.n_pod && !R.prio) || (R.n_out && !R.out)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "%s: unknown flags 0x%x", why ? name : "dra_preempt_batch", flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (max_victims && !victims) return fail(ctx, DRA_E_INVAL, "max_victims %u without a victims buffer", max_victims);
    if (budgets && budgets->n_pdb && !budgets->allowed)
        return fail(ctx, DRA_E_INVAL, "dra_preempt_pdb_batch: n_pdb %u without allowed", budgets->n_pdb);
    bool dense; uint32_t n_pair;
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_cands(ctx, n_pod, cand_nodes, cand_off, 0xFFFFFFFFu, ctx->n_node, 0xFFFFFFFFull, dense, n_pair)) ||
        (rc = check_sortable(ctx, n_pod ? R.n_pod : 0)) ||
        (rc = why_check(ctx, why, n_pair))) return rc;
    ctx->chain = why ? DRA_K_PREEMPT | DRA_K_UNSUITABLE_WHY : DRA_K_PREEMPT; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;
    if ((rc = check_budgets(ctx, "dra_preempt_pdb_batch", budgets, R.n_pod))) return rc;
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, std::max(n_claim, R.n_pod), 1, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    const size_t vb = (size_t)n_pod * max_victims * 4;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (!dense && (rc = grow_set(ctx, ctx->cap_pairs, (size_t)n_pair + 64, ctx->d_cand_nodes, ctx->d_pair_pod))) ||
        (rc = grow_set(ctx, ctx->cap_pre_pods, (size_t)n_pod + 8, ctx->d_pre_prio, ctx->d_pre_node, ctx->d_pre_nvic, ctx->d_pre_choice, ctx->d_pre_pst,
                       ctx->d_pre_podviol)) ||
        (rc = grow_set(ctx, ctx->cap_pre_pairs, (size_t)n_pair + 8, ctx->d_pre_psum, ctx->d_pre_psum64, ctx->d_pre_pairst, ctx->d_pre_pairvic,
                       ctx->d_pre_pairviol)) ||
        (rc = grow_set(ctx, ctx->cap_pre_vic, vb / 4 + 8, ctx->d_pre_vic))) return rc;
    const size_t np = why ? 0 : n_pod;                   // (the reasons call chooses nothing: no per-pod output)
    Outputs outs = {{pair_status, ctx->d_pre_pairst, pair_status ? (size_t)n_pair : 0},
                    {pair_victims, ctx->d_pre_pairvic, pair_victims ? (size_t)n_pair * 4 : 0},
                    {pod_node, ctx->d_pre_node, np * 4},
                    {pod_status, ctx->d_pre_pst, np},
                    {n_victims, ctx->d_pre_nvic, np * 4},
                    {victims, ctx->d_pre_vic, vb},
                    {pair_violations, ctx->d_pre_pairviol, pair_violations ? (size_t)n_pair * 4 : 0},
                    {pod_violations, ctx->d_pre_podviol, pod_violations ? (size_t)n_pod * 4 : 0}};
    if ((rc = why_buffers(ctx, why, outs, n_pair, n_pod, n_claim)) || (rc = reserve_out(ctx, outs))) return rc;
    Staging s;
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    s.add(ctx->d_pre_prio, prio, (size_t)n_pod * 4);
    if (!dense) {
        s.add(ctx->d_cand_off, cand_off, ((size_t)n_pod + 1) * 4);
        s.add(ctx->d_cand_nodes, cand_nodes, (size_t)n_pair * 4);
        s.add(ctx->d_pair_pod, nullptr, (size_t)n_pair * 4);
    }
    dra_running_pods Rd;
    dra_disruption_budgets Bd;
    if ((rc = running_parts(ctx, R, s, Rd, budgets, &Bd)) ||
        (rc = stage_in(ctx, s, [&](uint8_t* h) { expand_pairs((uint32_t*)h, cand_off, n_pod); }))) return rc;

    PreArgs a = pre_args(ctx, ctx->d_claims, ctx->d_pod_off, (const int32_t*)ctx->d_pre_prio, n_pod, dense ? nullptr : ctx->d_cand_nodes,
                         dense ? nullptr : ctx->d_cand_off, n_pair, Rd, ctx->d_inv_live, flags);
    a.pair_pod = dense ? nullptr : ctx->d_pair_pod;
    a.pair_status = pair_status ? ctx->d_pre_pairst : nullptr; a.pair_victims = pair_victims ? ctx->d_pre_pairvic : nullptr;
    a.n_victims = ctx->d_pre_nvic; a.choice = ctx->d_pre_choice; a.max_victims = max_victims;
    pre_budgets(ctx, a, budgets ? &Bd : nullptr);
    a.pair_viol = pair_violations ? ctx->d_pre_pairviol : nullptr; a.pod_viol = pod_violations ? ctx->d_pre_podviol : nullptr;
    Prof prof(ctx);
    if ((rc = launch_running_lists(ctx, a, prof, false))) return rc;
    const PreShard whole{0u, ctx->n_node, n_pair, 0u, nullptr, nullptr};   // every node: the walk index is the pair index
    if (why) {
        a.why = ctx->d_why; a.why_claim = ctx->d_why_claim;
        if ((rc = launch_preempt_pairs(ctx, a, whole, true)) ||
            (rc = launch_why_tally(ctx, *why, dense ? nullptr : ctx->d_cand_off, n_pod, n_claim))) return rc;
        prof.mark();
        return read_back(ctx, "preemption reasons kernels", 1, outs);
    }
    if ((rc = launch_preempt_pairs(ctx, a, whole))) return rc;
    cudaStream_t st = ctx->stream;
    k_pre_choose<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, st>>>(a);
    ctx->launches += 1;
    if (max_victims) {
        CU(cudaMemsetAsync(ctx->d_pre_vic, 0xFF, vb, st));
        launch_preempt_victims(ctx, a, ctx->d_pre_choice, 1u, ctx->d_pre_vic, max_victims);
    }
    prof.mark();
    return read_back(ctx, "preemption kernels", 1, outs);
}
}  // namespace

int dra_preempt_pdb_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, const int32_t* prio,
                          uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off, const dra_running_pods* running,
                          const dra_disruption_budgets* budgets, uint8_t* pair_status, uint32_t* pair_victims,
                          uint32_t* pair_violations, uint32_t* pod_node, uint8_t* pod_status, uint32_t* n_victims,
                          uint32_t* pod_violations, uint32_t* victims, uint32_t max_victims, uint32_t flags) {
    return preempt_call(ctx, "dra_preempt_pdb_batch", claims, n_claim, pod_off, prio, n_pod, cand_nodes, cand_off, running, budgets,
                        pair_status, pair_victims, pair_violations, pod_node, pod_status, n_victims, pod_violations, victims,
                        max_victims, nullptr, flags);
}

// Why preemption judged each node as it did (spec §19): dra_preempt_batch's pairs, each with its status, reason and
// blocking claim.  Budgets change no status and no reason, so the call takes none.
int dra_preempt_why_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, const int32_t* prio,
                          uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off, const dra_running_pods* running,
                          uint8_t* pair_status, uint8_t* pair_why, uint32_t* pair_claim, uint32_t* pod_why, uint32_t* claim_blocks,
                          uint32_t flags) {
    const WhyOut w{pair_why, pair_claim, pod_why, claim_blocks};
    return preempt_call(ctx, "dra_preempt_why_batch", claims, n_claim, pod_off, prio, n_pod, cand_nodes, cand_off, running, nullptr,
                        pair_status, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, &w, flags);
}

int dra_preempt_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, const int32_t* prio,
                      uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off, const dra_running_pods* running,
                      uint8_t* pair_status, uint32_t* pair_victims, uint32_t* pod_node, uint8_t* pod_status, uint32_t* n_victims,
                      uint32_t* victims, uint32_t max_victims, uint32_t flags) {
    return dra_preempt_pdb_batch(ctx, claims, n_claim, pod_off, prio, n_pod, cand_nodes, cand_off, running, nullptr, pair_status,
                                 pair_victims, nullptr, pod_node, pod_status, n_victims, nullptr, victims, max_victims, flags);
}

// Pod capacity (spec §16): every argument is checked here, before anything is staged or launched, so a rejected call
// writes nothing; the kernels read the live inventory and write only the call's own buffers.
int dra_pod_capacity_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off, uint32_t n_pod,
                           const uint32_t* cand_nodes, const uint32_t* cand_off, uint32_t max_copies, uint16_t* pair_copies,
                           uint8_t* pair_stop, uint64_t* pod_total, uint32_t* pod_nodes, uint32_t flags) {
    if (!ctx || !pod_off || (n_claim && !claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_pod_capacity_batch: unknown flags 0x%x", flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (max_copies < 1 || max_copies > 65535) return fail(ctx, DRA_E_INVAL, "max_copies %u outside [1, 65535]", max_copies);
    bool dense; uint32_t n_pair;
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_cands(ctx, n_pod, cand_nodes, cand_off, 0xFFFFFFFFu, ctx->n_node, 0xFFFFFFFFull, dense, n_pair))) return rc;
    if (n_pair && !pair_copies) return fail(ctx, DRA_E_INVAL, "pair_copies is NULL");
    ctx->chain = DRA_K_POD_CAPACITY; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, n_claim, 1, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (!dense && (rc = grow_set(ctx, ctx->cap_pairs, (size_t)n_pair + 64, ctx->d_cand_nodes, ctx->d_pair_pod))) ||
        (rc = grow_set(ctx, ctx->cap_cap_pairs, (size_t)n_pair + 8, ctx->d_cap_copies, ctx->d_cap_stop)) ||
        (rc = grow_set(ctx, ctx->cap_cap_pods, (size_t)n_pod + 8, ctx->d_cap_total, ctx->d_cap_nodes))) return rc;
    const Outputs outs = {{pair_copies, ctx->d_cap_copies, (size_t)n_pair * 2},
                          {pair_stop, ctx->d_cap_stop, pair_stop ? (size_t)n_pair : 0},
                          {pod_total, ctx->d_cap_total, pod_total ? (size_t)n_pod * 8 : 0},
                          {pod_nodes, ctx->d_cap_nodes, pod_nodes ? (size_t)n_pod * 4 : 0}};
    if ((rc = reserve_out(ctx, outs))) return rc;
    Staging s;
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    if (!dense) {
        s.add(ctx->d_cand_off, cand_off, ((size_t)n_pod + 1) * 4);
        s.add(ctx->d_cand_nodes, cand_nodes, (size_t)n_pair * 4);
        s.add(ctx->d_pair_pod, nullptr, (size_t)n_pair * 4);
    }
    if ((rc = stage_in(ctx, s, [&](uint8_t* h) { expand_pairs((uint32_t*)h, cand_off, n_pod); }))) return rc;
    CapArgs a; memset(&a, 0, sizeof a);
    a.claims = ctx->d_claims; a.pod_off = ctx->d_pod_off; a.n_pod = n_pod;
    a.cand_nodes = dense ? nullptr : ctx->d_cand_nodes; a.cand_off = dense ? nullptr : ctx->d_cand_off;
    a.pair_pod = dense ? nullptr : ctx->d_pair_pod; a.n_pair = n_pair;
    a.inv = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.tbl = ctx->d_tbl; a.sel = sel_of(ctx);
    a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u; a.max_copies = max_copies;
    a.node_lo = 0; a.n_win = ctx->n_node; a.n_walk = n_pair;           // every node: the walk index is the pair index
    a.pair_copies = ctx->d_cap_copies; a.pair_stop = pair_stop ? ctx->d_cap_stop : nullptr;
    a.pod_total = pod_total ? ctx->d_cap_total : nullptr; a.pod_nodes = pod_nodes ? ctx->d_cap_nodes : nullptr;
    Prof prof(ctx);
    if ((rc = launch_capacity(ctx, a))) return rc;
    prof.mark();
    return read_back(ctx, "capacity kernels", 1, outs);
}

// Preempt and place (spec §15): the pending-pod arrays are checked here, the running pods on the device (k_pre_running),
// whose fault gates the walk, so a rejected call writes no inventory word.  Running lists as in dra_preempt_batch (their
// offsets kept aside, since the visit lists reuse the sort's buffers), visit lists as in dra_place_pods_batch, then one
// persistent cooperative launch; the outputs are copied back after ONE synchronise and reach the caller only without a
// fault.  With why (spec §19, dra_preempt_place_why_batch) the walk is the reasons instantiation, k_pp_why_prep writes the
// pairs no walk reaches, and k_why_tally sums the records.
namespace {
int preempt_place_call(dra_ctx* ctx, const char* name, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off,
                       const int32_t* prio, uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off,
                       const dra_running_pods* running, const uint32_t* out_off, dra_out_rec* out, uint32_t n_out,
                       uint32_t* pod_node, uint8_t* pod_status, uint32_t* evicted_by, const WhyOut* why, uint8_t* pair_status,
                       uint32_t flags) {
    if (!ctx || !pod_off || !running || !running->pod_off || (n_claim && (!claims || !out)) ||
        (n_pod && (!prio || !pod_node || !pod_status)))
        return DRA_E_INVAL;
    const dra_running_pods& R = *running;
    if ((R.n_claim && !R.claims) || (R.n_pod && (!R.prio || !evicted_by)) || (R.n_out && !R.out)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "%s: unknown flags 0x%x", name, flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    bool dense; uint32_t n_pair;
    int rc;
    if ((rc = check_pod_off(ctx, pod_off, n_pod, n_claim)) ||
        (rc = check_cands(ctx, n_pod, cand_nodes, cand_off, PL_POS, ctx->n_node, 0xFFFFFFFFull, dense, n_pair))) return rc;
    if (!dense && n_pair > 0xFFFFFFF0u) return fail(ctx, DRA_E_INVAL, "too many (pod, node) pairs");   // (the dense form: below 2^32)
    if (ctx->n_node > PL_POS) return fail(ctx, DRA_E_INVAL, "more than %u nodes", PL_POS);
    if ((rc = check_slots(ctx, claims, n_claim, out_off, n_out, true)) ||
        (rc = check_sortable(ctx, n_pod ? R.n_pod : 0)) ||
        (rc = check_sortable(ctx, n_pod && !dense ? n_pair : 0)) ||
        (rc = why_check(ctx, why, n_pair))) return rc;
    ctx->chain = why ? DRA_K_PREEMPT_PLACE | DRA_K_PLACE_WHY : DRA_K_PREEMPT_PLACE; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;
    if (!ctx->coop_ok) return fail(ctx, DRA_E_STATE, "%s needs cooperative launches, which this device does not offer", name);
    CU(cudaSetDevice(ctx->device));
    if ((rc = ensure_batch(ctx, std::max(std::max(n_claim, R.n_pod), n_pair), n_out, true))) return rc;
    if ((rc = upload_table(ctx))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_pods, (size_t)n_pod + 8, ctx->d_pod_off, ctx->d_cand_off)) ||
        (!dense && (rc = grow_set(ctx, ctx->cap_pairs, (size_t)n_pair + 64, ctx->d_cand_nodes, ctx->d_pair_pod))) ||
        (rc = pp_buffers(ctx, n_pod, n_pair, R.n_pod))) return rc;
    const size_t rb = (size_t)n_out * 8;
    Outputs outs = {{out, ctx->d_out, rb}, {pod_node, ctx->d_pre_node, (size_t)n_pod * 4}, {pod_status, ctx->d_pre_pst, n_pod},
                    {evicted_by, ctx->d_pp_evicted, (size_t)R.n_pod * 4},
                    {pair_status, ctx->d_pre_pairst, pair_status ? (size_t)n_pair : 0}};
    if ((rc = why_buffers(ctx, why, outs, n_pair, n_pod, n_claim)) || (rc = reserve_out(ctx, outs))) return rc;
    Staging s;
    s.add(ctx->d_claims, claims, (size_t)n_claim * 16);
    s.add(ctx->d_pod_off, pod_off, ((size_t)n_pod + 1) * 4);
    if (out_off) s.add(ctx->d_out_off, out_off, (size_t)n_claim * 4);
    s.add(ctx->d_pre_prio, prio, (size_t)n_pod * 4);
    if (!dense) {
        s.add(ctx->d_cand_off, cand_off, ((size_t)n_pod + 1) * 4);
        s.add(ctx->d_cand_nodes, cand_nodes, (size_t)n_pair * 4);
    }
    dra_running_pods Rd;
    if ((rc = running_parts(ctx, R, s, Rd)) || (rc = stage_in(ctx, s))) return rc;
    cudaStream_t st = ctx->stream;
    if (rb) CU(cudaMemsetAsync(ctx->d_out, 0, rb, st));
    CU(cudaMemsetAsync(ctx->d_place_cursor, 0, ((size_t)ctx->n_node + 1) * 4, st));
    CU(cudaMemsetAsync(ctx->d_pp_judged, 0, ((size_t)ctx->n_node + 1) * 4, st));
    if (R.n_pod) CU(cudaMemsetAsync(ctx->d_pp_evicted, 0xFF, (size_t)R.n_pod * 4, st));

    PreArgs a = pre_args(ctx, ctx->d_claims, ctx->d_pod_off, (const int32_t*)ctx->d_pre_prio, n_pod, dense ? nullptr : ctx->d_cand_nodes,
                         dense ? nullptr : ctx->d_cand_off, n_pair, Rd, ctx->d_inv_live, flags);
    if (why) { a.pair_status = pair_status ? ctx->d_pre_pairst : nullptr; a.why = ctx->d_why; a.why_claim = ctx->d_why_claim; }
    Prof prof(ctx);
    if ((rc = launch_running_lists(ctx, a, prof, true))) return rc;
    // the visit lists (§13)
    PlaceArgs pl; memset(&pl, 0, sizeof pl);
    pl.claims = ctx->d_claims; pl.pod_off = ctx->d_pod_off; pl.n_pod = n_pod;
    pl.cand_nodes = a.cand_nodes; pl.cand_off = a.cand_off;
    pl.out_off = out_off ? ctx->d_out_off : nullptr; pl.out = ctx->d_out;
    pl.state = ctx->d_place_state; pl.pairs = ctx->d_podrec;
    pl.sorted = ctx->d_sorted; pl.list_off = ctx->d_claim_off; pl.cursor = ctx->d_place_cursor;
    pl.inv_src = ctx->d_inv_live; pl.inv_dst = ctx->d_inv_live; pl.node_off = ctx->d_node_off; pl.tbl = ctx->d_tbl;
    pl.n_node = ctx->n_node; pl.exhaustive = a.exhaustive; pl.sel = a.sel; pl.err = a.err;
    PpArgs pp{ctx->d_pp_pending, ctx->d_pp_evicted, ctx->d_pp_judged};
    k_pp_prep<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, st>>>(a, pl, pp);
    ctx->launches += 1;
    if (why) {
        k_pp_why_prep<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, st>>>(a, pl);
        ctx->launches += 1;
    }
    // A candidate form with no pair sorts nothing, so the visit lists are zeroed instead: the walk must not read the
    // offsets an earlier call's sort left in d_claim_off (an Allocate's claims by node), as lists of this call's pairs
    if (!dense && !n_pair) CU(cudaMemsetAsync(ctx->d_claim_off, 0, ((size_t)ctx->n_node + 2) * 4, st));
    if (!dense && n_pair &&
        (rc = launch_sort(ctx, ctx->d_podrec, n_pair, nullptr, nullptr, 0, 0, prof, ctx->d_inv_live, LA_NONE, ctx->n_node, ctx->d_node_off)))
        return rc;
    if (!why) {
        if ((rc = launch_walk(ctx, ctx->pp_occ, "k_pods_preempt_place", k_pods_preempt_place<4>, a, pl, pp))) return rc;
    } else {
        // (sized by its own occupancy: its registers are not k_pods_preempt_place<4>'s)
        if ((rc = launch_walk(ctx, ctx->pp_why_occ, "k_pods_preempt_place<4, true>", k_pods_preempt_place<4, true>, a, pl, pp)) ||
            (rc = launch_why_tally(ctx, *why, dense ? nullptr : ctx->d_cand_off, n_pod, n_claim)))
            return rc;
    }
    prof.mark();
    return read_back(ctx, why ? "preempt-and-place reasons kernels" : "preempt-and-place kernels", 1, outs);
}
}  // namespace

int dra_preempt_place_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off,
                            const int32_t* prio, uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off,
                            const dra_running_pods* running, const uint32_t* out_off, dra_out_rec* out, uint32_t n_out,
                            uint32_t* pod_node, uint8_t* pod_status, uint32_t* evicted_by, uint32_t flags) {
    return preempt_place_call(ctx, "dra_preempt_place_batch", claims, n_claim, pod_off, prio, n_pod, cand_nodes, cand_off, running,
                              out_off, out, n_out, pod_node, pod_status, evicted_by, nullptr, nullptr, flags);
}

// Why preemption judged each node as it did, in preempt and place (spec §19): dra_preempt_place_batch's call, every pair
// answered on the state its pod met
int dra_preempt_place_why_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* pod_off,
                                const int32_t* prio, uint32_t n_pod, const uint32_t* cand_nodes, const uint32_t* cand_off,
                                const dra_running_pods* running, const uint32_t* out_off, dra_out_rec* out, uint32_t n_out,
                                uint32_t* pod_node, uint8_t* pod_status, uint32_t* evicted_by, uint8_t* pair_status,
                                uint8_t* pair_why, uint32_t* pair_claim, uint32_t* pod_why, uint32_t* claim_blocks,
                                uint32_t flags) {
    const WhyOut w{pair_why, pair_claim, pod_why, claim_blocks};
    return preempt_place_call(ctx, "dra_preempt_place_why_batch", claims, n_claim, pod_off, prio, n_pod, cand_nodes, cand_off,
                              running, out_off, out, n_out, pod_node, pod_status, evicted_by, &w, pair_status, flags);
}

// Deallocate on one inventory (spec §9).  Every claim's slot range is checked here, with the slots k_dealloc counts, before
// anything is staged: k_dealloc applies each claim in its own thread, so a bad range found only on the device would leave
// the other claims' records applied.
int dra_deallocate_batch(dra_ctx* ctx, const dra_claim_rec* claims, uint32_t n_claim, const uint32_t* out_off,
                         const dra_out_rec* out, uint32_t n_out) {
    if (!ctx || (n_claim && (!claims || !out))) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (int rc = check_slots(ctx, claims, n_claim, out_off, n_out, false)) return rc;
    if (!n_claim) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_batch(ctx, n_claim, n_out, true);
    if (rc) return rc;
    const size_t cb = (size_t)n_claim * 16, ob = out_off ? (size_t)n_claim * 4 : 0, rb = (size_t)n_out * 8;
    if ((rc = grow_pinned(ctx, ctx->h_in, ctx->h_in_cap, cb + ob + rb))) return rc;
    memcpy(ctx->h_in, claims, cb);
    if (ob) memcpy(ctx->h_in + cb, out_off, ob);
    memcpy(ctx->h_in + cb + ob, out, rb);
    CU(cudaMemcpyAsync(ctx->d_claims, ctx->h_in, cb, cudaMemcpyHostToDevice, ctx->stream));
    if (ob) CU(cudaMemcpyAsync(ctx->d_out_off, ctx->h_in + cb, ob, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_out, ctx->h_in + cb + ob, rb, cudaMemcpyHostToDevice, ctx->stream));
    k_dealloc<<<(n_claim + 255) / 256, 256, 0, ctx->stream>>>(ctx->d_claims, n_claim, out_off ? ctx->d_out_off : nullptr,
                                                             ctx->d_out, n_out, (uint32_t*)ctx->d_inv_live, 0u, ctx->n_gpu, ctx->n_node,
                                                             nullptr, err_of(ctx));
    ctx->launches += 1;
    CU(cudaStreamSynchronize(ctx->stream));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "k_dealloc: %s", cudaGetErrorString(e));
    return check_err(ctx);
}

// ---- multi-GPU --------------------------------------------------------------------------------------

int dra_comm_unique_id(void* id128) {
    if (!id128) return DRA_E_INVAL;
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    std::string err;
    if (!g_nccl.load(err)) { g_create_err = err; return DRA_E_NCCL; }
    ncclUniqueId id;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclResult_t r = g_nccl.GetUniqueId(&id);
    if (r != ncclSuccess) { g_create_err = "ncclGetUniqueId failed"; return DRA_E_NCCL; }
    memcpy(id128, &id, 128);
    return DRA_OK;
}

int dra_comm_init(dra_ctx* ctx, const void* id128, int rank, int world) {
    if (!ctx || !id128 || world < 1 || rank < 0 || rank >= world) return DRA_E_INVAL;
    CU(cudaSetDevice(ctx->device));
    {
        std::lock_guard<std::mutex> lk(g_nccl_mu);
        std::string err;
        if (!g_nccl.load(err)) return fail(ctx, DRA_E_NCCL, "%s", err.c_str());
    }
    ncclUniqueId id; memcpy(&id, id128, 128);
    ncclResult_t r = g_nccl.CommInitRank(&ctx->comm, world, id, rank);
    if (r != ncclSuccess) return fail(ctx, DRA_E_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    ctx->rank = rank; ctx->world = world;
    return DRA_OK;
}

namespace {

// What a peer buffer's layout depends on.  Every rank computes its peers' offsets from its OWN layout, so an import requires
// every rank to be set up alike; the export writes this at offset 0 of the buffer for importers in other processes to read.
struct PeerLayout {
    uint32_t world, rank, form, cap, tab_len, inv_gpus;
    ShardSizes sizes;
    uint32_t pad;
    bool operator==(const PeerLayout& o) const { return memcmp(this, &o, sizeof o) == 0; }
};
PeerLayout layout_of(const dra_ctx* c, int rank) {
    PeerLayout l; memset(&l, 0, sizeof l);
    l.world = (uint32_t)c->world; l.rank = (uint32_t)rank; l.form = c->peer_form; l.cap = c->peer_cap; l.tab_len = c->peer_tab_len;
    l.inv_gpus = c->peer_inv_gpus; l.sizes = c->shard_rsv;
    return l;
}

using Kernels = std::initializer_list<const void*>;

// The counting sort's kernels (launch_sort), for the sharded chains that sort
const Kernels SORT_KERNELS = {(const void*)k_bucket_small, (const void*)k_bucket_hist8<false>, (const void*)k_bucket_hist8<true>,
                              (const void*)k_bucket_scan_rows, (const void*)k_bucket_scan8, (const void*)k_bucket_hist,
                              (const void*)k_bucket_scan, (const void*)k_bucket_scatter};

// Loads the kernels of a sharded chain now: ks, and waiting, those of its kernels that wait for its peers.  With lazy module
// loading (CUDA's default) the first launch of a kernel loads it, and the load waits for the kernels running on the
// device.  A rank's walk, merge or gather waits for its peers, so a host thread that enqueues the ranks of one process one
// after the other would stall at rank 0's first launch after such a kernel until the wait gives up.  Called while no call
// of the world is in flight.
// An SM holds CTAs of one L1/shared split at a time.  With ranks on one device, a rank's waiting kernels may sit on every
// SM while a peer's counting sort still has to run, and the sort's CTA-wide histogram wants most of the shared memory:
// the kernels that wait take the all-shared split, so the sort's CTAs fit beside them.
// sorts: the chain runs the counting sort.
int preload(dra_ctx* ctx, Kernels ks, Kernels waiting, bool sorts) {
    for (Kernels l : {ks, waiting, sorts ? SORT_KERNELS : Kernels{}})
        for (const void* k : l) { cudaFuncAttributes fa; CU(cudaFuncGetAttributes(&fa, k)); }
    for (const void* k : waiting) CU(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    return DRA_OK;
}

// uint4 units of one rank's pod-capacity slice for n walked pairs (dra_device.cuh CapMerge): the header, n u16 copies and
// n u8 stops, each padded to 16 bytes
size_t scap_units(uint32_t n) { return 1 + ((size_t)n + 7) / 8 + ((size_t)n + 15) / 16; }

// uint4 units of one rank's slice of the sharded reasons for n walked pairs (dra_device.cuh WhyMerge): the header, n u8
// reasons padded to 16 bytes, then (claims) n u32 blocking claims
size_t swhy_units(uint32_t n, bool claims = true) { return 1 + ((size_t)n + 15) / 16 + (claims ? ((size_t)n + 3) / 4 : 0); }

// The sharded preempt-and-place chain's kernels (preload), and the walk's occupancy query (which loads it too).  Its one
// wait is the inventory exchange (k_isync_copy), before the walk, and it keeps its split.
int preload_preempt_place_shard(dra_ctx* ctx) {
    if (int rc = preload(ctx, {(const void*)k_peer_push, (const void*)k_isync_copy, (const void*)k_spp_agree,
                               (const void*)k_pre_running, (const void*)k_pre_vsort, (const void*)k_spp_prep,
                               (const void*)k_pods_preempt_place<4>, (const void*)k_spp_final}, {}, true))
        return rc;
    if (ctx->pp_occ < 0) {
        int occ = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_pods_preempt_place<4>, 128, 0));
        ctx->pp_occ = occ;
    }
    return DRA_OK;
}

// The sharded preempt-and-place call's buffers for these sizes: the §15 walk's, the sort's, and the scratch inventory
int spp_buffers(dra_ctx* ctx, uint32_t n_pod, uint32_t n_pair, uint32_t rn_pod) {
    int rc;
    if ((rc = ensure_batch(ctx, std::max(std::max(rn_pod, n_pair), 1u), 1, false))) return rc;
    if ((rc = pp_buffers(ctx, n_pod, n_pair, rn_pod))) return rc;
    if ((rc = grow(ctx, ctx->d_spp_inv, ctx->cap_spp_inv, std::max(ctx->n_gpu, 1u)))) return rc;
    if (!ctx->d_spp_gate) CU(cudaMalloc((void**)&ctx->d_spp_gate, 16));
    return DRA_OK;
}

// uint4 units of one rank's preemption partials (dra_device.cuh PreShard): the header, n_pod partials of 2 + ceil(max_victims
// / 4) units, then n_pair {status, victims} pairs
size_t spre_units(uint32_t n_pod, uint32_t n_pair, uint32_t max_victims) {
    return 1 + (size_t)n_pod * (2 + ((size_t)max_victims + 3) / 4) + ((size_t)n_pair + 1) / 2;
}

// The sharded preemption call's own buffers for these sizes (the pair and running-pod groups as dra_preempt_batch grows them)
int spre_buffers(dra_ctx* ctx, uint32_t n_pod, uint32_t n_pair, uint32_t max_victims, uint32_t rn_pod) {
    int rc;
    if ((rc = grow(ctx, ctx->d_spre_part, ctx->cap_spre_part, spre_units(n_pod, n_pair, max_victims)))) return rc;
    if ((rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, std::max(n_pair, 1u)))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_pre_pairs, (size_t)n_pair + 8, ctx->d_pre_psum, ctx->d_pre_psum64, ctx->d_pre_pairst, ctx->d_pre_pairvic,
                       ctx->d_pre_pairviol)) ||
        (rc = grow_set(ctx, ctx->cap_pre_rpods, (size_t)rn_pod + 8, ctx->d_pre_rpodoff, ctx->d_pre_rprio, ctx->d_pre_rrec, ctx->d_pre_vlist,
                       ctx->d_pre_rpdb, ctx->d_pre_vprev))) return rc;
    return DRA_OK;
}

// (Re)allocates this rank's gather buffer:  [layout][table x2][staging x2: world slices of cap packets][headers x2][rendezvous flags]
// and, after dra_set_shard_pairs(max_pairs > 0), [UnsuitableNodes staging x2: world slices of uns_stride words][their flags]
// and, for dra_shard_export with an inventory loaded, [inventory staging x2: n_gpu records][their flags + election words]
// and, after dra_set_shard_place(max_pods > 0), [place pods: progress counter, 64 bytes][max_pods state words of 8 bytes]
// and, after dra_set_shard_preempt(max_pods > 0), [preemption partials x2: world slices of spre_units][their flags]
// and, after dra_set_shard_capacity(max_pairs > 0), [pod-capacity slices x2: world slices of scap_units][their flags]
// and, after dra_set_shard_why(max_pairs > 0), [reasons slices x2: world slices of swhy_units][their flags]
int peer_setup(dra_ctx* ctx, uint32_t form, uint32_t n_per, uint32_t tab_len, uint32_t cap) {
    if (ctx->world > (int)PEER_MAX) return fail(ctx, DRA_E_INVAL, "world %d > %u", ctx->world, PEER_MAX);
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->peer_ready = false;
    for (int r = 0; r < (int)PEER_MAX; ++r) {
        if (ctx->peer_base[r] && ctx->peer_ipc[r]) cudaIpcCloseMemHandle(ctx->peer_base[r]);
        ctx->peer_base[r] = nullptr; ctx->peer_ipc[r] = false;
    }
    if (ctx->peer_local) { CU(cudaFree(ctx->peer_local)); ctx->peer_local = nullptr; }
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
    auto reserve = [&](PeerRegion& rg, size_t stage_bytes, size_t slice, size_t flag_bytes) {   // stage_bytes 0: no staging
        if (stage_bytes) for (int p = 0; p < 2; ++p) rg.stage[p] = take(stage_bytes);
        rg.flags = take(flag_bytes); rg.slice = slice; rg.seq = 0;
    };
    take(sizeof(PeerLayout));                                                      // offset 0, whatever the sizes
    for (int p = 0; p < 2; ++p) ctx->off_table[p] = take((size_t)tab_len * 8 + 16);
    for (int p = 0; p < 2; ++p) ctx->off_stage[p] = take((size_t)ctx->world * cap * 16);
    for (int p = 0; p < 2; ++p) ctx->off_hdr[p] = take((size_t)ctx->world * 16);
    reserve(ctx->rendezvous_x, 0, 0, (size_t)PEER_MAX * 4);
    ctx->shard_rsv = ctx->shard_req;
    const ShardSizes& z = ctx->shard_rsv;
    ctx->uns_stride = (uint32_t)(((size_t)z.uns_pairs + 127) / 128 * 4);     // words, whole 16-byte units
    if (ctx->uns_stride) {
        reserve(ctx->uns_x, (size_t)ctx->world * ctx->uns_stride * 4, (size_t)ctx->uns_stride * 4, (size_t)PEER_MAX * 4);
        if (int rc = preload(ctx, {(const void*)k_uns_prep, (const void*)k_unsuitable<8, 8, false, true>,
                                   (const void*)k_unsuitable<8, 16, false, true>, (const void*)k_unsuitable<8, 32, false, true>,
                                   (const void*)k_unsuitable<8, 8, true, true>, (const void*)k_unsuitable<8, 16, true, true>,
                                   (const void*)k_unsuitable<8, 32, true, true>, (const void*)k_peer_push},
                             {(const void*)k_uns_merge}, false))
            return rc;
        // the call's own buffers at full size now: growing one inside the call would cudaFree the old one, which waits for
        // the whole device — where a peer's merge may already be spinning for this rank's push (ranks sharing a device)
        int rc;
        if ((rc = grow(ctx, ctx->d_ubits, ctx->cap_ubits, ctx->uns_stride))) return rc;
        if ((rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, z.uns_pairs))) return rc;
    }
    // the inventory sync's staging, sized for the inventory loaded now (sharded form only); its flags, then `elect` [2]
    ctx->peer_inv_gpus = form == 2 && ctx->d_inv_live ? ctx->n_gpu : 0u;
    if (ctx->peer_inv_gpus) reserve(ctx->isync_x, (size_t)ctx->peer_inv_gpus * 16, 0, (size_t)(PEER_MAX + 2) * 4);
    // sharded place pods, after dra_set_shard_place: the replicated state words (zeroed below, so the sequence starts over)
    if (z.place_pods) {
        ctx->off_splace = take(64 + (size_t)z.place_pods * 8);
        if (int rc = preload(ctx, {(const void*)k_splace_prep, (const void*)k_spod_gate, (const void*)k_splace_final},
                             {(const void*)k_pods_place<4, true>, (const void*)k_spod_gather<true>}, true))
            return rc;
        // the sort's scan-status words for the loaded inventory now: ensure_batch grows them with a cudaFree, which waits
        // for the whole device — where, inside a call, a peer's walk may be waiting for this rank
        if (ctx->d_inv_live) { if (int rc = ensure_batch(ctx, 1, 1, false)) return rc; }
    }
    // sharded preemption, after dra_set_shard_preempt: the partials' exchange, and the call's scratch at full size now (no
    // cudaFree inside a call while a peer's merge waits for this rank)
    if (z.pre_pods) {
        const size_t slice = spre_units(z.pre_pods, z.pre_pairs, z.pre_victims) * 16;
        reserve(ctx->pre_x, (size_t)ctx->world * slice, slice, (size_t)PEER_MAX * 4);
        if (int rc = preload(ctx, {(const void*)k_uns_prep, (const void*)k_pre_running, (const void*)k_pre_vsort,
                                   (const void*)k_pods_preempt<8, 8>, (const void*)k_pods_preempt<8, 16>,
                                   (const void*)k_pods_preempt<8, 32>, (const void*)k_spre_reduce,
                                   (const void*)k_pods_preempt_victims<8, 8>, (const void*)k_pods_preempt_victims<8, 16>,
                                   (const void*)k_pods_preempt_victims<8, 32>, (const void*)k_peer_push},
                             {(const void*)k_spre_merge}, true))
            return rc;
        if (int rc = spre_buffers(ctx, z.pre_pods, z.pre_pairs, z.pre_victims, 0)) return rc;
        if (ctx->d_inv_live) { if (int rc = ensure_batch(ctx, 1, 1, false)) return rc; }
    }
    // sharded pod capacity, after dra_set_shard_capacity: the slices' exchange, and the call's scratch at full size now (no
    // cudaFree inside a call while a peer's merge waits for this rank)
    if (z.scap_pairs) {
        const size_t slice = scap_units(z.scap_pairs) * 16;
        reserve(ctx->scap_x, (size_t)ctx->world * slice, slice, (size_t)PEER_MAX * 4);
        if (int rc = preload(ctx, {(const void*)k_uns_prep, (const void*)k_pods_capacity<8, 8>, (const void*)k_pods_capacity<8, 16>,
                                   (const void*)k_pods_capacity<8, 32>, (const void*)k_peer_push},
                             {(const void*)k_scap_merge}, false))
            return rc;
        if (int rc = grow(ctx, ctx->d_scap_part, ctx->cap_scap_part, scap_units(z.scap_pairs))) return rc;
        if (int rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, z.scap_pairs)) return rc;
    }
    // sharded reasons, after dra_set_shard_why: the slices' exchange (room for the claims: whether a call sends them is its
    // own choice), and the call's slice and pair -> pod at full size now (no cudaFree inside a call while a peer's merge
    // waits for this rank)
    if (z.swhy_pairs) {
        const size_t slice = swhy_units(z.swhy_pairs) * 16;
        reserve(ctx->swhy_x, (size_t)ctx->world * slice, slice, (size_t)PEER_MAX * 4);
        if (int rc = preload(ctx, {(const void*)k_uns_prep, (const void*)k_unsuitable<8, 8, false, true, true>,
                                   (const void*)k_unsuitable<8, 16, false, true, true>, (const void*)k_unsuitable<8, 32, false, true, true>,
                                   (const void*)k_unsuitable<8, 8, true, true, true>, (const void*)k_unsuitable<8, 16, true, true, true>,
                                   (const void*)k_unsuitable<8, 32, true, true, true>, (const void*)k_peer_push},
                             {(const void*)k_swhy_merge}, false))
            return rc;
        if (int rc = grow(ctx, ctx->d_swhy_part, ctx->cap_swhy_part, swhy_units(z.swhy_pairs))) return rc;
        if (int rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, z.swhy_pairs)) return rc;
    }
    // sharded place pods' reasons, after both reservations: the reasons walk and its prep loaded now (no module load
    // inside a call once a peer's walk may wait for this rank)
    if (z.place_pods && z.swhy_pairs) {
        if (int rc = preload(ctx, {(const void*)k_splace_why_prep}, {(const void*)k_pods_place<4, true, true>}, false)) return rc;
    }
    // sharded preempt and place, after dra_set_shard_preempt_place: its kernels loaded and its buffers at full size now (no
    // module load and no cudaFree inside a call while a peer's exchange waits for this rank)
    if (z.spp_pods) {
        reserve(ctx->spp_x, 0, 0, (size_t)PEER_MAX * 4);
        if (int rc = preload_preempt_place_shard(ctx)) return rc;
        if (ctx->d_inv_live) { if (int rc = spp_buffers(ctx, z.spp_pods, z.spp_pairs, z.spp_run)) return rc; }
        if (int rc = grow_set(ctx, ctx->cap_gtable, (size_t)tab_len + 16, ctx->d_gtable)) return rc;   // the call's table, at the exported size
    }
    ctx->splace_seq = 0;
    if (ctx->d_splace_local) CU(cudaMemset(ctx->d_splace_local, 0, 64 + ctx->cap_splace_local * 8));
    ctx->peer_bytes = off;
    CU(cudaMalloc((void**)&ctx->peer_local, ctx->peer_bytes));
    CU(cudaMemset(ctx->peer_local, 0, ctx->peer_bytes));
    if (!ctx->d_cursor) CU(cudaMalloc((void**)&ctx->d_cursor, 64));
    CU(cudaMemset(ctx->d_cursor, 0, 64));
    ctx->peer_form = form; ctx->peer_n_per = n_per; ctx->peer_tab_len = tab_len; ctx->peer_cap = cap; ctx->peer_epoch = 0;
    const PeerLayout mine = layout_of(ctx, ctx->rank);
    CU(cudaMemcpy(ctx->peer_local, &mine, sizeof mine, cudaMemcpyHostToDevice));
    if (const char* e = getenv("DRA_PEER_TIMEOUT_MS")) ctx->peer_spin = std::max(1ll, atoll(e)) * 1900000ll;
    ctx->gather_table = nullptr;
    ctx->state_epoch++;
    return DRA_OK;
}

PktGather make_gather(dra_ctx* ctx, uint32_t epoch, uint32_t slot_base, uint32_t n_per, uint32_t count, const uint32_t* count_dev) {
    PktGather g; memset(&g, 0, sizeof g);
    const uint32_t par = epoch & 1u;
    for (int r = 0; r < ctx->world; ++r) {
        g.stage[r] = (uint4*)(ctx->peer_base[r] + ctx->off_stage[par]) + (size_t)ctx->rank * ctx->peer_cap;
        g.hdr[r] = (uint4*)(ctx->peer_base[r] + ctx->off_hdr[par]) + ctx->rank;
    }
    g.my_stage = (const uint4*)(ctx->peer_local + ctx->off_stage[par]);
    g.my_hdr = (const uint4*)(ctx->peer_local + ctx->off_hdr[par]);
    g.table = (uint2*)(ctx->peer_local + ctx->off_table[par]);
    g.cursor = ctx->d_cursor;
    g.world = ctx->world; g.rank = ctx->rank; g.cap = ctx->peer_cap; g.epoch = epoch; g.parity = par;
    g.slot_base = slot_base; g.n_per = n_per; g.count = count; g.count_dev = count_dev; g.spin_limit = ctx->peer_spin;
    return g;
}

// The next call of the exchange whose region is rg
PeerExchange bind_exchange(dra_ctx* ctx, PeerRegion& rg) {
    PeerExchange x; memset(&x, 0, sizeof x);
    x.world = (uint32_t)ctx->world; x.rank = (uint32_t)ctx->rank; x.seq = ++rg.seq; x.spin_limit = ctx->peer_spin; x.err = err_of(ctx);
    const size_t stage = rg.stage[x.seq & 1u];
    for (int r = 0; r < ctx->world; ++r) {
        x.stage[r] = (uint4*)(ctx->peer_base[r] + stage + (size_t)ctx->rank * rg.slice);
        x.flag[r] = (uint32_t*)(ctx->peer_base[r] + rg.flags) + ctx->rank;
    }
    x.my_stage = (const uint4*)(ctx->peer_local + stage);
    x.my_flags = (const uint32_t*)(ctx->peer_local + rg.flags);
    return x;
}

// The next call of the exchange whose region is rg, with this rank's n4 units at src pushed to every peer (k_peer_push).
// World 1 (no gather): no peers, nothing pushed.
PeerExchange push_slice(dra_ctx* ctx, PeerRegion& rg, bool gather, const uint4* src, uint32_t n4) {
    if (!gather) return PeerExchange{};
    const PeerExchange x = bind_exchange(ctx, rg);
    k_peer_push<<<push_grid(ctx, n4), 256, 0, ctx->stream>>>(x, src, 0u, n4);
    ctx->launches += 1;
    return x;
}

// The first kernel of the sharded pair calls (k_uns_prep): pod_off and cand_off (nullptr: dense form) checked, and in the
// candidate form pair -> pod into d_upair_pod.  Its fault gates the pair kernel.
void launch_uns_prep(dra_ctx* ctx, const uint32_t* d_pod_off, const uint32_t* d_cand_off, uint32_t n_pod, uint32_t n_claim,
                     uint32_t n_pair) {
    k_uns_prep<<<std::max(1u, (n_pod + 7) / 8), 256, 0, ctx->stream>>>(d_pod_off, d_cand_off, n_pod, n_claim, n_pair,
                                                                       ctx->d_upair_pod, err_of(ctx));
    ctx->launches += 1;
}

// A merge's shard bounds: rank r owns nodes [bounds[r], bounds[r + 1]); world 1 (no gather): every node
void merge_bounds(const dra_ctx* ctx, bool gather, uint32_t (&bounds)[PEER_MAX + 1]) {
    bounds[0] = 0; bounds[1] = ctx->n_node;
    if (gather) for (int r = 0; r <= ctx->world; ++r) bounds[r] = ctx->shard_bounds[r];
}

// The sharded reasons' exchange at world > 1 (check_world's reserved()): dra_set_shard_why before the export, since even a
// call with no pairs pushes a header and raises flags, which would land in the peers' buffers at offset 0
int swhy_reserved(dra_ctx* ctx) {
    if (ctx->shard_rsv.swhy_pairs) return DRA_OK;
    return fail(ctx, DRA_E_STATE, "world > 1: dra_set_shard_why(max_pairs > 0) was not called before dra_shard_export");
}

// n_why answered pairs within the sharded reasons' exchange (check_world's fits())
int swhy_fits(dra_ctx* ctx, uint32_t n_why) {
    if (n_why <= ctx->shard_rsv.swhy_pairs) return DRA_OK;
    return fail(ctx, DRA_E_INVAL, "%u pairs exceed the max_pairs (%u) of dra_set_shard_why before dra_shard_export", n_why,
                ctx->shard_rsv.swhy_pairs);
}

// The sharded reasons' buffers, grown before the call enqueues anything else: this rank's slice for n_walk walked pairs
// (world > 1: peer_setup sized it for max_pairs, which bounds n_walk, so it never reallocates there) and, with
// claim_blocks, the merge's per-claim counts, zeroed.  Those depend on n_claim, which no setter bounds: a larger batch grows
// them here, the old buffer retired until the next dra_ctx_sync.
int swhy_buffers(dra_ctx* ctx, const WhyOut& w, uint32_t n_walk, uint32_t n_claim) {
    if (int rc = grow(ctx, ctx->d_swhy_part, ctx->cap_swhy_part, swhy_units(n_walk))) return rc;
    if (!w.claim_blocks) return DRA_OK;
    if (int rc = grow(ctx, ctx->d_swhy_blocks, ctx->cap_swhy_blocks, (size_t)n_claim + 1)) return rc;
    CU(cudaMemsetAsync(ctx->d_swhy_blocks, 0, ((size_t)n_claim + 1) * 4, ctx->stream));
    return DRA_OK;
}

// Where the walk writes its reasons in this rank's slice: [header][n_walk u8 reasons, padded][n_walk u32 claims].  The
// claims are written whether they are sent or not.
void swhy_slice(const dra_ctx* ctx, uint32_t n_walk, uint8_t*& why, uint32_t*& why_claim) {
    why = reinterpret_cast<uint8_t*>(ctx->d_swhy_part + 1);
    why_claim = reinterpret_cast<uint32_t*>(ctx->d_swhy_part + 1 + ((size_t)n_walk + 15) / 16);
}

// After the walk: this rank's slice to every rank behind its header, the fault word at gate (push_slice advances the
// region's call parity, as every §17 call does), then the owner-indexed merge writes w's outputs and the tallies on every
// rank (k_swhy_merge).  cand_nodes and cand_off: nullptr in the dense form.  Enqueues only.
int launch_swhy_merge(dra_ctx* ctx, const WhyOut& w, const uint32_t* gate, uint32_t n_walk, const uint32_t* cand_nodes,
                      const uint32_t* cand_off, uint32_t n_pod, uint32_t n_pair, uint32_t n_claim) {
    const bool gather = ctx->world > 1;
    uint4* part = ctx->d_swhy_part;
    WhyMerge m; memset(&m, 0, sizeof m);
    m.part = part; m.cand_nodes = cand_nodes; m.cand_off = cand_off;
    m.n_pod = n_pod; m.n_pair = n_pair; m.n_node = ctx->n_node; m.n_claim = n_claim;
    merge_bounds(ctx, gather, m.bounds);
    m.gate = gate;
    m.pair_why = w.pair_why; m.pair_claim = w.pair_claim; m.pod_why = w.pod_why; m.claim_blocks = w.claim_blocks;
    m.blocks = ctx->d_swhy_blocks;
    if (gather) {
        m.slice4 = (uint32_t)(ctx->swhy_x.slice / 16);
        CU(cudaMemcpyAsync(part, gate, 4, cudaMemcpyDeviceToDevice, ctx->stream));   // the header: this rank's fault word
    }
    const PeerExchange x = push_slice(ctx, ctx->swhy_x, gather, part, (uint32_t)swhy_units(n_walk, w.pair_claim || w.claim_blocks));
    k_swhy_merge<<<wait_grid(ctx, (n_pod + 7) / 8), 256, 0, ctx->stream>>>(x, m);
    ctx->launches += 1;
    return DRA_OK;
}

// The result table of a global Allocate call: at world > 1 the table of g, a gather of a new epoch, else this context's own
int result_table(dra_ctx* ctx, uint32_t n_out, const uint32_t* count_dev, PktGather& g, uint2*& table) {
    if (ctx->world > 1) {
        ctx->peer_epoch += 1;
        g = make_gather(ctx, ctx->peer_epoch, 0, 0, 0, count_dev);
    } else if (int rc = grow_set(ctx, ctx->cap_gtable, (size_t)n_out + 16, ctx->d_gtable)) {
        return rc;
    }
    table = ctx->world > 1 ? g.table : ctx->d_gtable;
    return DRA_OK;
}

// A sharded call's claims and OutRec slots: at most 2^26 of each, and without out_off one slot per claim at least
int check_slots(dra_ctx* ctx, uint32_t n_claim, uint32_t n_out, bool have_off) {
    if (n_claim > (1u << 26) || n_out > (1u << 26)) return fail(ctx, DRA_E_INVAL, "batch too large for the sharded call (2^26)");
    if (!have_off && n_out < n_claim) return fail(ctx, DRA_E_INVAL, "n_out %u < n_claim %u without out_off", n_out, n_claim);
    return DRA_OK;
}

int launch_gather(dra_ctx* ctx, const PktGather& g, const uint4* d_claims, uint32_t n_claim, const uint32_t* n_dev,
                  const uint32_t* d_out_off, uint32_t n_out, uint32_t have_off, uint32_t n_node) {
    const uint32_t blocks = std::max(1u, std::min((uint32_t)ctx->n_sm * 2u, (std::max(n_claim, g.world * g.cap / 4u) + 255u) / 256u));
    k_pkt_gather<<<blocks, 256, 0, ctx->stream>>>(g, d_claims, n_claim, n_dev, d_out_off, n_out, have_off, n_node, err_of(ctx));
    ctx->launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "k_pkt_gather: %s", cudaGetErrorString(e));
    return DRA_OK;
}

}  // namespace

int dra_peer_export(dra_ctx* ctx, uint32_t n_per_rank, void* handle64) {
    if (!ctx) return DRA_E_INVAL;
    if (!n_per_rank) { ctx->peer_ready = false; return DRA_OK; }          // switch the peer path off (NCCL again)
    if (!handle64) return DRA_E_INVAL;
    int rc = peer_setup(ctx, 1, n_per_rank, (uint32_t)ctx->world * n_per_rank, n_per_rank);
    if (rc) return rc;
    cudaIpcMemHandle_t h;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    CU(cudaIpcGetMemHandle(&h, ctx->peer_local));
    memcpy(handle64, &h, 64);
    return DRA_OK;
}

int dra_shard_export(dra_ctx* ctx, uint32_t n_out_max, uint32_t cap_per_rank, void* handle64) {
    if (!ctx || !n_out_max) return DRA_E_INVAL;
    if (n_out_max > (1u << 26)) return fail(ctx, DRA_E_INVAL, "n_out_max %u exceeds 2^26", n_out_max);
    int rc = peer_setup(ctx, 2, 0, n_out_max, cap_per_rank ? std::min(cap_per_rank, n_out_max) : n_out_max);
    if (rc) return rc;
    if (handle64) {
        cudaIpcMemHandle_t h;
        CU(cudaIpcGetMemHandle(&h, ctx->peer_local));
        memcpy(handle64, &h, 64);
    }
    return DRA_OK;
}

int dra_peer_import(dra_ctx* ctx, const void* handles) {
    if (!ctx || !handles) return DRA_E_INVAL;
    if (!ctx->peer_local) return fail(ctx, DRA_E_STATE, "dra_peer_export / dra_shard_export has not been called");
    CU(cudaSetDevice(ctx->device));
    for (int r = 0; r < ctx->world; ++r) {
        if (r == ctx->rank) { ctx->peer_base[r] = ctx->peer_local; ctx->peer_ipc[r] = false; continue; }
        cudaIpcMemHandle_t h; memcpy(&h, (const uint8_t*)handles + (size_t)r * 64, 64);
        void* p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(ctx, DRA_E_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e)); }
        ctx->peer_base[r] = (uint8_t*)p; ctx->peer_ipc[r] = true;
        // a peer laid out differently would take this rank's stores at offsets past its regions: refuse it here
        PeerLayout theirs;
        CU(cudaMemcpy(&theirs, p, sizeof theirs, cudaMemcpyDeviceToHost));
        if (!(theirs == layout_of(ctx, r))) return fail(ctx, DRA_E_INVAL, "dra_peer_import: rank %d is not set up like this one", r);
    }
    ctx->peers_on_device = 1;
    ctx->peer_ready = true;
    return DRA_OK;
}

int dra_peer_import_local(dra_ctx* ctx, dra_ctx* const* ctxs) {
    if (!ctx || !ctxs) return DRA_E_INVAL;
    if (!ctx->peer_local) return fail(ctx, DRA_E_STATE, "dra_peer_export / dra_shard_export has not been called");
    CU(cudaSetDevice(ctx->device));
    for (int r = 0; r < ctx->world; ++r) {
        dra_ctx* o = ctxs[r];
        if (!o || !o->peer_local || o->rank != r || !(layout_of(o, r) == layout_of(ctx, r)))
            return fail(ctx, DRA_E_INVAL, "dra_peer_import_local: context %d is not set up like this one", r);
        if (o->device != ctx->device) {
            int ok = 0; CU(cudaDeviceCanAccessPeer(&ok, ctx->device, o->device));
            if (!ok) return fail(ctx, DRA_E_CUDA, "no peer access from device %d to %d", ctx->device, o->device);
            cudaError_t e = cudaDeviceEnablePeerAccess(o->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(ctx, DRA_E_CUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e));
            (void)cudaGetLastError();
        }
        ctx->peer_base[r] = o->peer_local; ctx->peer_ipc[r] = false;
    }
    ctx->peers_on_device = 0;
    for (int r = 0; r < ctx->world; ++r) ctx->peers_on_device += ctxs[r]->device == ctx->device ? 1 : 0;
    ctx->peer_ready = true;
    return DRA_OK;
}

int dra_peer_rendezvous_device(dra_ctx* ctx) {
    if (!ctx) return DRA_E_INVAL;
    QUIESCE();
    if (ctx->world <= 1) return DRA_OK;
    if (!ctx->peer_ready) return fail(ctx, DRA_E_STATE, "dra_peer_import has not been called");
    CU(cudaSetDevice(ctx->device));
    k_rendezvous<<<1, 32, 0, ctx->stream>>>(bind_exchange(ctx, ctx->rendezvous_x));   // (not counted in dra_launch_count: it is no part of a batch)
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "k_rendezvous: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int dra_comm_init_local(dra_ctx* ctx, int rank, int world) {
    if (!ctx || world < 1 || world > (int)PEER_MAX || rank < 0 || rank >= world) return DRA_E_INVAL;
    ctx->rank = rank; ctx->world = world;
    return DRA_OK;
}

int dra_allocate_batch_gather_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim, const uint32_t* d_out_off,
                                     dra_out_rec* d_out_all, uint32_t n_out, uint32_t n_per_rank, uint32_t flags) {
    if (!ctx || (n_claim && !d_claims)) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->comm && !ctx->peer_ready) return fail(ctx, DRA_E_STATE, "dra_comm_init has not been called");
    if (!d_out_all && !ctx->peer_ready) return fail(ctx, DRA_E_INVAL, "d_out_all may be NULL only with the peer all-gather set up");
    if (n_out > n_per_rank) return fail(ctx, DRA_E_INVAL, "n_out %u > n_per_rank %u", n_out, n_per_rank);
    ctx->chain = ctx->chain_tile = 0;
    CU(cudaSetDevice(ctx->device));
    int rc = ensure_batch(ctx, n_claim, n_out, false);
    if (rc) return rc;

    if (ctx->peer_ready && ctx->peer_form == 1 && n_per_rank == ctx->peer_n_per) {
        // ---- packet all-gather over NVLink: rides in the tail of the fused kernel, or runs as its own kernel ----
        ctx->peer_epoch += 1;
        const PktGather g = make_gather(ctx, ctx->peer_epoch, (uint32_t)ctx->rank * n_per_rank, n_per_rank, n_out, nullptr);
        uint2* mine = g.table + g.slot_base;
        bool tail_done = false;
        rc = launch_allocate(ctx, (const uint4*)d_claims, n_claim, d_out_off, mine, n_out, flags, &g, &tail_done);
        if (rc) return rc;
        if (!tail_done && (rc = launch_gather(ctx, g, (const uint4*)d_claims, n_claim, nullptr, d_out_off, n_out, d_out_off != nullptr, ctx->n_node))) return rc;
        ctx->gather_table = (const dra_out_rec*)g.table; ctx->gather_n_per = n_per_rank; ctx->gather_len = 0;
        if (d_out_all) CU(cudaMemcpyAsync(d_out_all, g.table, (size_t)ctx->world * n_per_rank * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        if (ctx->profiling && !tail_done) { cudaEventRecord(ctx->ev[5], ctx->stream); ctx->ev_mask |= 1u << 5; }
        return DRA_OK;
    }

    if (!ctx->comm) return fail(ctx, DRA_E_STATE, "dra_comm_init has not been called (NCCL path)");
    if (!d_out_all) return fail(ctx, DRA_E_INVAL, "d_out_all is required on the NCCL path");
    ctx->gather_table = d_out_all; ctx->gather_n_per = n_per_rank; ctx->gather_len = 0;
    dra_out_rec* mine = d_out_all + (size_t)ctx->rank * n_per_rank;
    if (n_per_rank > n_out) CU(cudaMemsetAsync(mine + n_out, 0, (size_t)(n_per_rank - n_out) * 8, ctx->stream));
    rc = launch_allocate(ctx, (const uint4*)d_claims, n_claim, d_out_off, (uint2*)mine, n_out, flags);
    if (rc) return rc;
    // the one collective of the path: every rank's OutRec slice to every rank (in place), same stream
    ncclResult_t r = g_nccl.AllGather(mine, d_out_all, (size_t)n_per_rank * 8, ncclUint8, ctx->comm, ctx->stream);
    if (r != ncclSuccess) return fail(ctx, DRA_E_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    if (ctx->profiling) { cudaEventRecord(ctx->ev[5], ctx->stream); ctx->ev_mask |= 1u << 5; }
    return DRA_OK;
}

// ---- sharded global batch -------------------------------------------------------------------------------

int dra_set_shard(dra_ctx* ctx, uint32_t node_lo, uint32_t node_hi, int take_stray) {
    if (!ctx) return DRA_E_INVAL;
    if (node_lo > node_hi || node_hi > ctx->n_node) return fail(ctx, DRA_E_INVAL, "shard [%u, %u) outside the inventory's %u nodes", node_lo, node_hi, ctx->n_node);
    CU(cudaSetDevice(ctx->device));
    CU(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_sc_counts) ctx->h_sc_counts[3] = 0u;           // a new partition: the old call's count is no plan hint any more
    ctx->shard_on = true; ctx->shard_lo = node_lo; ctx->shard_hi = node_hi; ctx->shard_stray = take_stray ? 1u : 0u;
    ctx->shard_map_on = false;
    ctx->state_epoch++;
    return DRA_OK;
}

int dra_set_shard_map(dra_ctx* ctx, const uint32_t* bounds, int stray_rank) {
    if (!ctx || !bounds) return DRA_E_INVAL;
    if (stray_rank < 0 || stray_rank >= ctx->world) return fail(ctx, DRA_E_INVAL, "stray_rank %d outside the world of %d", stray_rank, ctx->world);
    if (bounds[0] != 0 || bounds[ctx->world] != ctx->n_node) return fail(ctx, DRA_E_INVAL, "shard map must span [0, %u]", ctx->n_node);
    for (int r = 0; r < ctx->world; ++r) if (bounds[r + 1] < bounds[r]) return fail(ctx, DRA_E_INVAL, "shard map not monotone at rank %d", r);
    int rc = dra_set_shard(ctx, bounds[ctx->rank], bounds[ctx->rank + 1], stray_rank == ctx->rank);
    if (rc) return rc;
    for (int r = 0; r <= ctx->world; ++r) ctx->shard_bounds[r] = bounds[r];
    ctx->shard_stray_rank = (uint32_t)stray_rank; ctx->shard_map_on = true;
    return DRA_OK;
}

int dra_allocate_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim, const uint32_t* d_out_off,
                                     uint32_t n_out, uint32_t flags) {
    if (!ctx || (n_claim && !d_claims)) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (flags & ~DRA_F_FRESH_INVENTORY) return fail(ctx, DRA_E_INVAL, "dra_allocate_batch_global_device: unsupported flags 0x%x", flags);
    if (int rc = check_slots(ctx, n_claim, n_out, d_out_off != nullptr)) return rc;
    const bool gather = ctx->world > 1;
    if (int rc = need_peers(ctx)) return rc;
    if (gather && n_out > ctx->peer_tab_len) return fail(ctx, DRA_E_INVAL, "n_out %u exceeds the exported table (%u)", n_out, ctx->peer_tab_len);
    ctx->chain = ctx->chain_tile = 0;
    // world > 1: a peer on this device may already be waiting for this rank's packets, so a buffer this call outgrows
    // is freed at the next dra_ctx_sync (a cudaFree now would wait for that peer, which waits for this call)
    CallScope scope{ctx};
    if (int rc = scope.open(gather)) return rc;
    const uint32_t n_local_node = ctx->shard_hi - ctx->shard_lo;
    // Plan.  The single-launch kernel lays its shared memory out for a CAPACITY of claims; the real number is only known
    // on the device (the compaction's count).  First call of a shape: capacity = the whole batch (always safe).  Later
    // calls: the last completed call's count plus slack — as much slack as still lets the claim array be STAGED in shared
    // memory (the fast form).  If more claims than the capacity fall into the shard the kernel touches nothing, tells its
    // peers, and the call fails with DRA_E_STATE ("call again": the next plan uses the new count).
    uint32_t cap = n_claim;
    FusedPlan plan = fused_plan(ctx, cap, flags, n_local_node);
    if (ctx->h_sc_counts && ctx->h_sc_counts[3] != 0u && ctx->shard_last_n == n_claim) {
        const uint32_t expect = ctx->h_sc_counts[0];
        const uint32_t hi = (uint32_t)std::min<uint64_t>(n_claim, (uint64_t)expect + expect / 4 + 256);
        const uint32_t lo = (uint32_t)std::min<uint64_t>(n_claim, (uint64_t)expect + expect / 32 + 64);
        FusedPlan ph = fused_plan(ctx, hi, flags, n_local_node);
        cap = hi; plan = ph;
        if (ph.fused && !ph.stage) {                            // shrink the slack until the array fits shared memory
            for (uint32_t c = hi; c >= lo; c -= std::max(1u, (hi - lo) / 16u)) {
                const FusedPlan pc = fused_plan(ctx, c, flags, n_local_node);
                if (pc.fused && pc.stage) { cap = c; plan = pc; break; }
                if (c == lo || c - lo < std::max(1u, (hi - lo) / 16u)) {
                    const FusedPlan pl = fused_plan(ctx, lo, flags, n_local_node);
                    if (pl.fused && pl.stage) { cap = lo; plan = pl; }
                    break;
                }
            }
        }
    }
    if (!plan.fused) cap = n_claim;                           // sort path: no layout depends on the count
    ctx->shard_last_n = n_claim;
    int rc = ensure_batch(ctx, std::max(cap, 1u), n_out, false);
    if (rc) return rc;
    if ((rc = grow_set(ctx, ctx->cap_cclaims, (size_t)n_claim + 64, ctx->d_cclaims, ctx->d_coff))) return rc;
    // tiles: 256 claims while that keeps them within 1024 (one round of predecessor reads), else 2048; beyond 2M claims
    // the look-back kernel
    const uint32_t sc_rows = n_claim <= 256u * 1024u ? 1u : 8u;
    const bool sc_flat = n_claim <= 2048u * 1024u;
    const uint32_t n_tiles = std::max(1u, (n_claim + 256u * sc_rows - 1) / (256u * sc_rows));
    if ((size_t)n_tiles + 8 > ctx->cap_sc_status) {
        const size_t ncap = (size_t)n_tiles * 2 + 64;
        if ((rc = grow_nc(ctx, ctx->d_sc_status, 0, ncap))) return rc;
        CU(cudaMemsetAsync(ctx->d_sc_status, 0, ncap * 8, ctx->stream));
        ctx->cap_sc_status = ncap;
    }
    if (!ctx->d_sc_counts) {
        CU(cudaMalloc((void**)&ctx->d_sc_counts, 64)); CU(cudaMemsetAsync(ctx->d_sc_counts, 0, 64, ctx->stream));
        void* hp = nullptr;
        CU(cudaHostAlloc(&hp, 64, cudaHostAllocMapped));
        memset(hp, 0, 64);
        ctx->h_sc_counts = (volatile uint32_t*)hp;
        CU(cudaHostGetDevicePointer((void**)&ctx->h_sc_counts_dev, hp, 0));
    }
    if (!ctx->d_rank_slots) { CU(cudaMalloc((void**)&ctx->d_rank_slots, 2 * PEER_MAX * 4)); CU(cudaMemsetAsync(ctx->d_rank_slots, 0, 2 * PEER_MAX * 4, ctx->stream)); }
    const bool counted = gather && ctx->shard_map_on;          // every rank counts every rank's slots: the gather needs no header
    uint2* table = nullptr; PktGather g; memset(&g, 0, sizeof g);
    if ((rc = result_table(ctx, n_out, ctx->d_sc_counts + 1, g, table))) return rc;
    // 1. this rank's claims, compacted in input order, node indices local to the shard
    ctx->shard_epoch += 1;
    // A tile takes a predecessor's status word for this call's when the word's 10-bit epoch matches and its state is set, so a
    // word left 1,024 calls back would pass.  The call whose epoch wraps to 0 starts from cleared words — all of them, since a
    // later call may have more tiles than this one — and no word older than that call can then alias.
    if ((ctx->shard_epoch & 0x3FFu) == 0u) CU(cudaMemsetAsync(ctx->d_sc_status, 0, ctx->cap_sc_status * 8, ctx->stream));
    if (counted) g.expect = ctx->d_rank_slots + (ctx->shard_epoch & 1u) * PEER_MAX;
    ShardArgs sa; memset(&sa, 0, sizeof sa);
    if (counted) {
        sa.world = (uint32_t)ctx->world; sa.stray_rank = ctx->shard_stray_rank; sa.rank_slots = ctx->d_rank_slots;
        for (int r = 0; r < ctx->world; ++r) sa.rank_hi[r] = ctx->shard_bounds[r + 1];
    }
    sa.claims = (const uint4*)d_claims; sa.n_claim = n_claim; sa.out_off = d_out_off;
    sa.node_lo = ctx->shard_lo; sa.node_hi = ctx->shard_hi; sa.n_node_global = ctx->n_node; sa.take_stray = ctx->shard_stray;
    sa.have_off = d_out_off != nullptr;
    sa.cclaims = ctx->d_cclaims; sa.coff = ctx->d_coff; sa.cap = (uint32_t)std::min<size_t>(ctx->cap_cclaims, 0xFFFFFFFFu);
    sa.status = ctx->d_sc_status; sa.ticket = ctx->d_ticket + TK_COMPACT; sa.n_tiles = n_tiles; sa.epoch = ctx->shard_epoch;
    sa.counts = ctx->d_sc_counts; sa.h_counts = ctx->h_sc_counts_dev; sa.err = err_of(ctx);
    if (getenv("DRA_TIMELINE")) {                              // instrumentation: two words, read back with dra_debug_shard_times
        if (!ctx->d_sc_times) CU(cudaMalloc((void**)&ctx->d_sc_times, 16));
        const unsigned long long init[2] = {~0ull, 0ull};
        CU(cudaMemcpyAsync(ctx->d_sc_times, init, 16, cudaMemcpyHostToDevice, ctx->stream));
        sa.timeline = ctx->d_sc_times;
    }
    // (launched by launch_allocate, right before the kernel that reads the list)
    // 2. the usual chain on the shard's view of the inventory, results at the claims' GLOBAL slots
    AllocView view; view.node_lo = ctx->shard_lo; view.n_node = n_local_node; view.n_dev = ctx->d_sc_counts; view.have_off = d_out_off != nullptr;
    view.sa = &sa; view.sc_rows = sc_rows; view.sc_flat = sc_flat;
    bool tail_done = false;
    rc = launch_allocate(ctx, ctx->d_cclaims, cap, ctx->d_coff, table, n_out, flags, gather ? &g : nullptr, &tail_done, &view);
    if (rc) return rc;
    if (gather && !tail_done && (rc = launch_gather(ctx, g, ctx->d_cclaims, cap, ctx->d_sc_counts, ctx->d_coff, n_out, d_out_off != nullptr, n_local_node))) return rc;
    ctx->gather_table = (const dra_out_rec*)table; ctx->gather_n_per = n_out; ctx->gather_len = n_out;
    return DRA_OK;
}

int dra_set_shard_pairs(dra_ctx* ctx, uint32_t max_pairs) {
    if (!ctx) return DRA_E_INVAL;
    if (int rc = check_before_export(ctx, "dra_set_shard_pairs")) return rc;
    if (max_pairs > 0xFFFFFFF0u) return fail(ctx, DRA_E_INVAL, "max_pairs %u: too many (pod, node) pairs", max_pairs);
    ctx->shard_req.uns_pairs = max_pairs;
    return DRA_OK;
}

// Sharded UnsuitableNodes: prep (offset checks, pair -> pod) -> k_unsuitable on this rank's node window -> push of this rank's
// words to every peer -> wait + OR into the caller's bytes.  Enqueues only.
int dra_unsuitable_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                       const uint32_t* d_pod_off, uint32_t n_pod,
                                       const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                       uint8_t* d_suitable_bits, uint32_t flags) {
    if (!ctx || !d_pod_off || (n_claim && !d_claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_unsuitable_batch_global_device: unknown flags 0x%x", flags);
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    bool dense;
    if (int rc = check_dev_cands(ctx, d_cand_nodes, d_cand_off, n_pod, n_pair, true, dense)) return rc;
    const bool gather = ctx->world > 1;
    const uint32_t max_pairs = ctx->shard_rsv.uns_pairs;
    if (int rc = check_world(ctx, nullptr, false, no_check, -1, [&] {
            if (n_pair <= max_pairs) return (int)DRA_OK;
            return fail(ctx, DRA_E_INVAL, "n_pair %u exceeds the max_pairs (%u) of dra_set_shard_pairs before dra_shard_export", n_pair, max_pairs);
        }))
        return rc;
    if (n_pair && !d_suitable_bits) return DRA_E_INVAL;
    if (!n_pair) return DRA_OK;                        // every rank sees the same n_pair: none of them exchanges anything
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    const size_t n_words = ((size_t)n_pair + 31) / 32, n_words4 = ((size_t)n_pair + 127) / 128 * 4;
    // world > 1: peer_setup sized both for max_pairs, so these never reallocate there (no cudaFree while peers wait)
    if ((rc = grow(ctx, ctx->d_ubits, ctx->cap_ubits, n_words4))) return rc;
    if (!dense && (rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, n_pair))) return rc;
    CU(cudaMemsetAsync(ctx->d_ubits, 0, n_words4 * 4, ctx->stream));
    launch_uns_prep(ctx, d_pod_off, d_cand_off, n_pod, n_claim, n_pair);
    UnsArgs a; memset(&a, 0, sizeof a);
    a.claims = (const uint4*)d_claims; a.pod_off = d_pod_off; a.n_pod = n_pod;
    a.cand_nodes = d_cand_nodes; a.cand_off = d_cand_off; a.pair_pod = ctx->d_upair_pod;
    a.inv = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.tbl = ctx->d_tbl; a.bits = ctx->d_ubits;
    a.sel = sel_of(ctx);
    a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u;
    a.node_lo = ctx->shard_lo; a.n_win = ctx->shard_hi - ctx->shard_lo;
    a.n_walk = dense ? n_pod * a.n_win : n_pair;           // (n_pod * n_win <= n_pod * n_node = n_pair)
    a.gate = ctx->d_err + ERR_BAD_OFFSETS;
    Prof prof(ctx);
    if (a.n_walk && (rc = launch_unsuitable(ctx, a, true))) return rc;
    prof.mark();
    UnsMerge m; memset(&m, 0, sizeof m);
    m.bits = ctx->d_ubits; m.out = d_suitable_bits;
    m.n_words = (uint32_t)n_words; m.n_bytes = (uint32_t)(((size_t)n_pair + 7) / 8); m.stride = ctx->uns_stride;
    const PeerExchange x = push_slice(ctx, ctx->uns_x, gather, (const uint4*)ctx->d_ubits, (uint32_t)(n_words4 / 4));
    k_uns_merge<<<wait_grid(ctx, (n_words + 1023) / 1024), 256, 0, ctx->stream>>>(x, m);
    ctx->launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded UnsuitableNodes launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

// Sharded pods Allocate: pod records + ownership over every pod (k_spod_records) -> gate / FRESH copy (k_spod_gate) ->
// stable counting sort of this rank's pods by window node -> k_pods on the window -> all-gather of the owned pods' records
// (k_spod_gather).  Enqueues only.
int dra_allocate_pods_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                          const uint32_t* d_pod_off, uint32_t n_pod,
                                          const uint32_t* d_out_off, uint32_t n_out, uint32_t flags) {
    if (!ctx || !d_pod_off || (n_claim && !d_claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~(DRA_F_EXHAUSTIVE | DRA_F_FRESH_INVENTORY))
        return fail(ctx, DRA_E_INVAL, "dra_allocate_pods_batch_global_device: unknown flags 0x%x", flags);
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (n_pod > (1u << 26)) return fail(ctx, DRA_E_INVAL, "batch too large for the sharded call (2^26)");
    if (int rc = check_slots(ctx, n_claim, n_out, d_out_off != nullptr)) return rc;
    if (!n_pod && n_claim) return fail(ctx, DRA_E_INVAL, "pod_off must span [0, n_claim]: no pods for %u claims", n_claim);
    const bool gather = ctx->world > 1;
    if (int rc = check_world(ctx, "the gather needs", false, no_check, n_out, no_check)) return rc;
    ctx->chain = ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;                         // every rank sees the same n_pod: none of them exchanges anything
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    const uint32_t n_win = ctx->shard_hi - ctx->shard_lo;
    if ((rc = ensure_batch(ctx, n_pod, 1, false))) return rc;
    const Tiling t = tiling(n_pod, n_win, ctx->n_sm);                 // the sort's tiles are laid out on the window
    if ((rc = grow(ctx, ctx->d_hist, ctx->cap_hist, (size_t)t.n_tiles * (n_win + 1), 64))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_podrec, (size_t)n_pod + 8, ctx->d_podrec))) return rc;
    if (!ctx->d_spod) CU(cudaMalloc((void**)&ctx->d_spod, SP_WORDS * 4));
    uint2* table = nullptr; PktGather g; memset(&g, 0, sizeof g);
    if ((rc = result_table(ctx, n_out, nullptr, g, table))) return rc;
    if (gather) g.expect = ctx->d_spod + SP_EXPECT;
    const Err err = err_of(ctx);
    SPodArgs sa; memset(&sa, 0, sizeof sa);
    sa.claims = (const uint4*)d_claims; sa.pod_off = d_pod_off; sa.out_off = d_out_off;
    sa.n_claim = n_claim; sa.n_pod = n_pod; sa.n_out = n_out; sa.n_node = ctx->n_node;
    sa.node_lo = ctx->shard_lo; sa.node_hi = ctx->shard_hi; sa.take_stray = ctx->shard_stray;
    sa.rank = (uint32_t)ctx->rank; sa.world = gather ? (uint32_t)ctx->world : 1u; sa.stray_rank = ctx->shard_stray_rank;
    if (gather) for (int r = 0; r < ctx->world; ++r) sa.rank_hi[r] = ctx->shard_bounds[r + 1];
    sa.table = table; sa.podrec = ctx->d_podrec; sa.w = ctx->d_spod; sa.err = err;
    const bool fresh = (flags & DRA_F_FRESH_INVENTORY) != 0;
    Prof prof(ctx);
    CU(cudaMemsetAsync(ctx->d_spod, 0, (SP_BAD + 1) * 4, ctx->stream));
    k_spod_records<<<(n_pod + 255) / 256, 256, 0, ctx->stream>>>(sa);
    const uint32_t gate_grid = fresh ? std::max(1u, std::min((uint32_t)ctx->n_sm, (ctx->n_gpu + 255) / 256)) : 1u;
    k_spod_gate<<<gate_grid, 256, 0, ctx->stream>>>(sa, gather ? ctx->peer_cap : 0u, fresh ? ctx->d_inv_pristine : nullptr,
                                                    ctx->d_inv_live, ctx->d_node_off);
    ctx->launches += 2; ctx->chain |= DRA_K_POD_SHARD;
    const uint32_t* d_node_off = ctx->d_node_off + ctx->shard_lo;
    if ((rc = launch_sort(ctx, ctx->d_podrec, n_pod, nullptr, nullptr, 0, 0, prof, ctx->d_inv_live, LA_NONE, n_win, d_node_off,
                          ctx->d_spod + SP_NDEV))) return rc;
    if (n_win) {
        PodArgs a; memset(&a, 0, sizeof a);
        a.claims = (const uint4*)d_claims; a.out_off = d_out_off; a.out = table;
        a.sorted = ctx->d_sorted; a.claim_off = ctx->d_claim_off;
        a.inv_src = ctx->d_inv_live; a.inv_dst = ctx->d_inv_live; a.node_off = d_node_off; a.tbl = ctx->d_tbl;
        a.n_node = n_win; a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u; a.sel = sel_of(ctx); a.err = err;
        const uint32_t grid = std::max(1u, std::min((n_win + 3) / 4, (uint32_t)ctx->n_sm * 8u));
        CU(launch_k(k_pods<4>, dim3(grid), dim3(128), 0, ctx->stream, pdl_attr(ctx), a));
        ctx->launches += 1;
    }
    prof.mark();
    if (gather) {
        k_spod_gather<false><<<wait_grid(ctx, (std::max(n_pod, g.world * g.cap / 4u) + 255u) / 256u), 256, 0, ctx->stream>>>(g, sa, ctx->peer_tab_len);
        ctx->launches += 1; ctx->chain |= DRA_K_POD_GATHER;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded pods Allocate launch: %s", cudaGetErrorString(e));
    ctx->gather_table = (const dra_out_rec*)table; ctx->gather_n_per = n_out; ctx->gather_len = n_out;
    return DRA_OK;
}

int dra_set_shard_place(dra_ctx* ctx, uint32_t max_pods) {
    if (!ctx) return DRA_E_INVAL;
    if (int rc = check_before_export(ctx, "dra_set_shard_place")) return rc;
    if (max_pods > (1u << 26)) return fail(ctx, DRA_E_INVAL, "max_pods %u exceeds 2^26", max_pods);
    ctx->shard_req.place_pods = max_pods;
    return DRA_OK;
}

// Sharded place pods: checks, initial state words, pair records and every rank's slot bound (k_splace_prep) -> gate / FRESH
// copy (k_spod_gate) -> stable counting sort of the pairs by window node -> the persistent walk of the window's visit lists,
// every state word published to every rank (k_pods_place<4, true>) -> pod_node and the finalisers' slots (k_splace_final) ->
// expected counts (k_spod_gate) -> all-gather of the finalised pods' records (k_spod_gather<true>).  Enqueues only.
// With why (spec §18, dra_place_pods_why_batch_global_device): the reasons walk k_pods_place<4, true, true> writes this
// rank's slice of §17's sharded exchange at the walk index, k_splace_why_prep (after the gate) the window's pairs no walk
// reaches, and after the gather the slice goes to every peer behind its header — the walk's fault word, set when the call
// is gated or the walk timed out — and k_swhy_merge writes the four reason outputs on every rank.
namespace {
int place_pods_shard_call(dra_ctx* ctx, const char* name, const dra_claim_rec* d_claims, uint32_t n_claim,
                          const uint32_t* d_pod_off, uint32_t n_pod, const uint32_t* d_cand_nodes, const uint32_t* d_cand_off,
                          uint32_t n_pair, const uint32_t* d_out_off, uint32_t n_out, uint32_t* d_pod_node, const WhyOut* why,
                          uint32_t flags) {
    if (!ctx || !d_pod_off || (n_claim && !d_claims) || (n_pod && !d_pod_node)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~(DRA_F_EXHAUSTIVE | DRA_F_FRESH_INVENTORY))
        return fail(ctx, DRA_E_INVAL, "%s: unknown flags 0x%x", name, flags);
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (n_pod > (1u << 26)) return fail(ctx, DRA_E_INVAL, "batch too large for the sharded call (2^26)");
    if (int rc = check_slots(ctx, n_claim, n_out, d_out_off != nullptr)) return rc;
    if (!n_pod && n_claim) return fail(ctx, DRA_E_INVAL, "pod_off must span [0, n_claim]: no pods for %u claims", n_claim);
    bool dense;
    if (int rc = check_dev_cands(ctx, d_cand_nodes, d_cand_off, n_pod, n_pair, false, dense)) return rc;
    if (ctx->n_node > PL_POS) return fail(ctx, DRA_E_INVAL, "more than %u nodes", PL_POS);
    uint32_t n_why;
    if (int rc = place_why_pairs(ctx, why, dense, n_pod, n_pair, n_why)) return rc;
    const bool gather = ctx->world > 1;
    const uint32_t max_pods = ctx->shard_rsv.place_pods;
    if (int rc = check_world(ctx, "the walk and the gather need", false, [&] { return why ? swhy_reserved(ctx) : (int)DRA_OK; },
                             n_out, [&] {
            if (n_pod > max_pods)
                return fail(ctx, DRA_E_STATE, "n_pod %u exceeds the max_pods (%u) of dra_set_shard_place before dra_shard_export", n_pod, max_pods);
            return swhy_fits(ctx, n_why);
        }))
        return rc;
    if (int rc = why_check(ctx, why, n_why)) return rc;
    ctx->chain = ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;                         // every rank sees the same n_pod: none of them exchanges anything
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    const uint32_t n_win = ctx->shard_hi - ctx->shard_lo;
    const uint32_t n_walk = dense ? n_pod * n_win : n_pair;           // (n_pod * n_win <= n_pod * n_node < 2^32)
    // (the blocks are zeroed here, before the walk: after it, this thread launches only kernels peer_setup preloaded)
    if (why && (rc = swhy_buffers(ctx, *why, n_walk, n_claim))) return rc;
    if ((rc = ensure_batch(ctx, std::max(n_pod, n_pair), 1, false))) return rc;
    const Tiling t = tiling(n_pair, n_win, ctx->n_sm);                // the sort's tiles are laid out on the window
    if ((rc = grow(ctx, ctx->d_hist, ctx->cap_hist, (size_t)t.n_tiles * (n_win + 1), 64))) return rc;
    if ((rc = grow_set(ctx, ctx->cap_podrec, (size_t)n_pair + 8, ctx->d_podrec)) ||
        (rc = grow(ctx, ctx->d_splace_rec, ctx->cap_splace_rec, n_pod)) ||
        (rc = grow_set(ctx, ctx->cap_place_cursor, (size_t)n_win + 8, ctx->d_place_cursor))) return rc;
    if (!gather && n_pod > ctx->cap_splace_local) {          // world 1: the state words in plain device memory, zeroed
        const size_t cap = (size_t)n_pod + n_pod / 2 + 64;
        if (ctx->d_splace_local) CU(cudaFree(ctx->d_splace_local));
        ctx->d_splace_local = nullptr;
        CU(cudaMalloc((void**)&ctx->d_splace_local, 64 + cap * 8));
        CU(cudaMemsetAsync(ctx->d_splace_local, 0, 64 + cap * 8, ctx->stream));
        ctx->cap_splace_local = cap;
    }
    if (!ctx->d_spod) CU(cudaMalloc((void**)&ctx->d_spod, SP_WORDS * 4));
    uint2* table = nullptr; PktGather g; memset(&g, 0, sizeof g);
    if ((rc = result_table(ctx, n_out, nullptr, g, table))) return rc;
    if (gather) g.expect = ctx->d_spod + SP_EXPECT;
    const Err err = err_of(ctx);
    const bool fresh = (flags & DRA_F_FRESH_INVENTORY) != 0;
    const uint32_t* d_node_off = ctx->d_node_off + ctx->shard_lo;

    PlaceShard sh; memset(&sh, 0, sizeof sh);
    for (int r = 0; r < (gather ? ctx->world : 1); ++r) {
        uint8_t* base = gather ? ctx->peer_base[r] + ctx->off_splace : ctx->d_splace_local;
        sh.prog[r] = (uint32_t*)base; sh.rep[r] = (unsigned long long*)(base + 64);
    }
    sh.gated = ctx->d_spod + SP_GATED; sh.w = ctx->d_spod; sh.podrec = ctx->d_splace_rec;
    sh.world = gather ? (uint32_t)ctx->world : 1u; sh.rank = gather ? (uint32_t)ctx->rank : 0u; sh.seq = ++ctx->splace_seq;
    sh.node_lo = ctx->shard_lo; sh.n_win = n_win;
    sh.n_claim = n_claim; sh.n_pair = n_pair; sh.n_out = n_out;
    for (uint32_t r = 0; r < sh.world; ++r) sh.rank_hi[r] = gather ? ctx->shard_bounds[r + 1] : ctx->n_node;
    sh.spin_limit = ctx->peer_spin;
    PlaceArgs a; memset(&a, 0, sizeof a);
    a.claims = (const uint4*)d_claims; a.pod_off = d_pod_off; a.n_pod = n_pod;
    a.cand_nodes = dense ? nullptr : d_cand_nodes; a.cand_off = dense ? nullptr : d_cand_off;
    a.out_off = d_out_off; a.out = table; a.pod_node = d_pod_node; a.pairs = ctx->d_podrec;
    a.sorted = ctx->d_sorted; a.list_off = ctx->d_claim_off; a.cursor = ctx->d_place_cursor;
    a.inv_src = ctx->d_inv_live; a.inv_dst = ctx->d_inv_live; a.node_off = d_node_off; a.tbl = ctx->d_tbl;
    a.n_node = ctx->n_node; a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u; a.sel = sel_of(ctx); a.err = err;
    if (why) swhy_slice(ctx, n_walk, a.why, a.why_claim);
    // the gate's SPodArgs: its record count is the sort's (the pairs), its world the one the bounds were counted for
    SPodArgs sa; memset(&sa, 0, sizeof sa);
    sa.claims = (const uint4*)d_claims; sa.pod_off = d_pod_off; sa.out_off = d_out_off;
    sa.n_claim = n_claim; sa.n_pod = n_pod; sa.n_out = n_out; sa.n_node = ctx->n_node;
    sa.node_lo = ctx->shard_lo; sa.node_hi = ctx->shard_hi; sa.rank = sh.rank; sa.world = sh.world;
    sa.table = table; sa.podrec = ctx->d_splace_rec; sa.w = ctx->d_spod; sa.err = err;
    SPodArgs sa_sort = sa; sa_sort.n_pod = dense ? 0u : n_pair;

    Prof prof(ctx);
    CU(cudaMemsetAsync(ctx->d_spod, 0, (SP_BAD + 1) * 4, ctx->stream));
    if (n_out) CU(cudaMemsetAsync(table, 0, (size_t)n_out * 8, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_place_cursor, 0, ((size_t)n_win + 1) * 4, ctx->stream));
    if (why) CU(cudaMemsetAsync(ctx->d_spod + SP_WHY_FAULT, 0, 4, ctx->stream));
    k_splace_prep<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, ctx->stream>>>(a, sh);
    const uint32_t gate_grid = fresh ? std::max(1u, std::min((uint32_t)ctx->n_sm, (ctx->n_gpu + 255) / 256)) : 1u;
    k_spod_gate<<<gate_grid, 256, 0, ctx->stream>>>(sa_sort, gather ? ctx->peer_cap : 0u, fresh ? ctx->d_inv_pristine : nullptr,
                                                    ctx->d_inv_live, ctx->d_node_off);
    ctx->launches += 2;
    if (why) {
        k_splace_why_prep<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, ctx->stream>>>(a, sh);
        ctx->launches += 1;
    }
    // A candidate form with no pair sorts nothing, so the visit lists are zeroed instead: the walk must not read the
    // offsets an earlier call's sort left in d_claim_off (an Allocate's claims by node), as lists of this call's pairs
    if (!dense && !n_pair) CU(cudaMemsetAsync(ctx->d_claim_off, 0, ((size_t)ctx->n_node + 2) * 4, ctx->stream));
    if (!dense && n_pair && n_win &&
        (rc = launch_sort(ctx, ctx->d_podrec, n_pair, nullptr, nullptr, 0, 0, prof, ctx->d_inv_live, LA_NONE, n_win, d_node_off,
                          ctx->d_spod + SP_NDEV)))
        return rc;
    // The gate has read the bounds: k_splace_final counts the slots each rank really finalises in the same words.  (Zeroed
    // before the walk: after it, this thread launches only kernels peer_setup preloaded, since anything it waits for there
    // would hold back the peers' calls that the walk waits for.)
    CU(cudaMemsetAsync(ctx->d_spod, 0, PEER_MAX * 4, ctx->stream));
    // Every CTA resident, not a cooperative launch: cooperative grids do not run beside each other, and a rank's walk waits
    // for its peers' walks
    if (!why) {
        if ((rc = walk_occupancy(ctx, ctx->splace_occ, "k_pods_place<4, true>", k_pods_place<4, true>))) return rc;
        k_pods_place<4, true><<<shard_walk_grid(ctx, ctx->splace_occ, gather, n_win), 128, 0, ctx->stream>>>(a, sh);
    } else {
        // (sized by its own occupancy: its registers are not k_pods_place<4, true>'s)
        if ((rc = walk_occupancy(ctx, ctx->splace_why_occ, "k_pods_place<4, true, true>", k_pods_place<4, true, true>))) return rc;
        k_pods_place<4, true, true><<<shard_walk_grid(ctx, ctx->splace_why_occ, gather, n_win), 128, 0, ctx->stream>>>(a, sh);
    }
    ctx->launches += 1;
    k_splace_final<<<(n_pod + 255) / 256, 256, 0, ctx->stream>>>(a, sh);
    ctx->launches += 1; ctx->chain |= DRA_K_PLACE_SHARD;
    prof.mark();
    if (gather) {
        k_spod_gate<<<1, 256, 0, ctx->stream>>>(sa, ctx->peer_cap, nullptr, ctx->d_inv_live, ctx->d_node_off);
        k_spod_gather<true><<<wait_grid(ctx, (std::max(n_pod, g.world * g.cap / 4u) + 255u) / 256u), 256, 0, ctx->stream>>>(g, sa, ctx->peer_tab_len);
        ctx->launches += 2;
    }
    if (why) {
        // the gate: the walk's fault word
        if ((rc = launch_swhy_merge(ctx, *why, ctx->d_spod + SP_WHY_FAULT, n_walk, a.cand_nodes, a.cand_off, n_pod, n_pair, n_claim)))
            return rc;
        ctx->chain |= DRA_K_PLACE_WHY;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "%s launch: %s", why ? "sharded place reasons" : "sharded place pods", cudaGetErrorString(e));
    ctx->gather_table = (const dra_out_rec*)table; ctx->gather_n_per = n_out; ctx->gather_len = n_out;
    return DRA_OK;
}
}  // namespace

int dra_place_pods_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                       const uint32_t* d_pod_off, uint32_t n_pod,
                                       const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                       const uint32_t* d_out_off, uint32_t n_out, uint32_t* d_pod_node, uint32_t flags) {
    return place_pods_shard_call(ctx, "dra_place_pods_batch_global_device", d_claims, n_claim, d_pod_off, n_pod, d_cand_nodes,
                                 d_cand_off, n_pair, d_out_off, n_out, d_pod_node, nullptr, flags);
}

// Why place pods put each pod where it did, across a sharded world (spec §18 "Sharded form")
int dra_place_pods_why_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                           const uint32_t* d_pod_off, uint32_t n_pod,
                                           const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                           const uint32_t* d_out_off, uint32_t n_out, uint32_t* d_pod_node,
                                           uint8_t* d_pair_why, uint32_t* d_pair_claim, uint32_t* d_pod_why,
                                           uint32_t* d_claim_blocks, uint32_t flags) {
    const WhyOut w{d_pair_why, d_pair_claim, d_pod_why, d_claim_blocks};
    return place_pods_shard_call(ctx, "dra_place_pods_why_batch_global_device", d_claims, n_claim, d_pod_off, n_pod,
                                 d_cand_nodes, d_cand_off, n_pair, d_out_off, n_out, d_pod_node, &w, flags);
}

int dra_set_shard_preempt(dra_ctx* ctx, uint32_t max_pods, uint32_t max_pairs, uint32_t max_victims) {
    if (!ctx) return DRA_E_INVAL;
    if (int rc = check_before_export(ctx, "dra_set_shard_preempt")) return rc;
    if (max_pods > (1u << 26) || max_pairs > 0xFFFFFFF0u || max_victims > (1u << 20))
        return fail(ctx, DRA_E_INVAL, "dra_set_shard_preempt: sizes too large (max_pods <= 2^26, max_victims <= 2^20)");
    if (spre_units(max_pods, max_pairs, max_victims) > ((size_t)1 << 32) / 16)
        return fail(ctx, DRA_E_INVAL, "dra_set_shard_preempt: one rank's slice would exceed 4 GiB");
    ShardSizes& z = ctx->shard_req;
    z.pre_pods = max_pods; z.pre_pairs = max_pairs; z.pre_victims = max_victims;
    return DRA_OK;
}

// Sharded preemption: offset checks and pair -> pod (k_uns_prep) -> the running pods, their bucketing and victim lists on
// the whole inventory (k_pre_running, the counting sort, k_pre_vsort) -> the window's pairs (k_pods_preempt) -> per-pod
// partials (k_spre_reduce, k_pods_preempt_victims) -> push to every peer -> wait + merge into the caller's buffers (k_spre_merge).
// Enqueues only.
int dra_preempt_pdb_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                        const uint32_t* d_pod_off, const int32_t* d_prio, uint32_t n_pod,
                                        const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                        const dra_running_pods* running, const dra_disruption_budgets* budgets,
                                        uint8_t* d_pair_status, uint32_t* d_pair_victims, uint32_t* d_pair_violations,
                                        uint32_t* d_pod_node, uint8_t* d_pod_status, uint32_t* d_n_victims,
                                        uint32_t* d_pod_violations, uint32_t* d_victims, uint32_t max_victims, uint32_t flags) {
    if (!ctx || !d_pod_off || !running || !running->pod_off || (n_claim && !d_claims) ||
        (n_pod && (!d_prio || !d_pod_node || !d_pod_status || !d_n_victims)))
        return DRA_E_INVAL;
    const dra_running_pods& R = *running;
    if ((R.n_claim && !R.claims) || (R.n_pod && !R.prio) || (R.n_out && !R.out)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_preempt_batch_global_device: unknown flags 0x%x", flags);
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (max_victims && !d_victims) return fail(ctx, DRA_E_INVAL, "max_victims %u without a victims buffer", max_victims);
    if (budgets && budgets->n_pdb && !budgets->allowed)
        return fail(ctx, DRA_E_INVAL, "dra_preempt_pdb_batch_global_device: n_pdb %u without allowed", budgets->n_pdb);
    bool dense;
    if (int rc = check_dev_cands(ctx, d_cand_nodes, d_cand_off, n_pod, n_pair, true, dense)) return rc;
    if (n_pod > (1u << 26) || max_victims > (1u << 20)) return fail(ctx, DRA_E_INVAL, "n_pod or max_victims too large for the sharded call");
    const bool gather = ctx->world > 1;
    const ShardSizes& z = ctx->shard_rsv;
    if (int rc = check_world(ctx, "the merge needs", true, no_check, -1, [&] {
            if (n_pod <= z.pre_pods && n_pair <= z.pre_pairs && max_victims <= z.pre_victims) return (int)DRA_OK;
            return fail(ctx, DRA_E_INVAL, "n_pod %u / n_pair %u / max_victims %u exceed the sizes of dra_set_shard_preempt before dra_shard_export "
                        "(%u / %u / %u)", n_pod, n_pair, max_victims, z.pre_pods, z.pre_pairs, z.pre_victims);
        }))
        return rc;
    ctx->chain = DRA_K_PREEMPT_SHARD; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;                         // every rank sees the same n_pod: none of them exchanges anything
    if (int rc = check_budgets(ctx, "dra_preempt_pdb_batch_global_device", budgets, R.n_pod)) return rc;
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    if ((rc = ensure_batch(ctx, std::max(R.n_pod, 1u), 1, false))) return rc;
    if ((rc = spre_buffers(ctx, n_pod, n_pair, max_victims, R.n_pod))) return rc;
    cudaStream_t st = ctx->stream;
    const uint32_t lo = gather ? ctx->shard_lo : 0u, hi = gather ? ctx->shard_hi : ctx->n_node;   // world 1: every node
    const bool want_pairs = d_pair_status || d_pair_victims || d_pair_violations;
    PreShard s; memset(&s, 0, sizeof s);
    s.node_lo = lo; s.n_win = hi - lo; s.n_walk = dense ? n_pod * s.n_win : n_pair;
    s.stride = 2 + (max_victims + 3) / 4; s.part = ctx->d_spre_part;
    s.pairs = want_pairs ? reinterpret_cast<uint2*>(ctx->d_spre_part + 1 + (size_t)n_pod * s.stride) : nullptr;

    PreArgs a = pre_args(ctx, (const uint4*)d_claims, d_pod_off, d_prio, n_pod, dense ? nullptr : d_cand_nodes,
                         dense ? nullptr : d_cand_off, n_pair, R, ctx->d_inv_live, flags);
    a.pair_pod = dense ? nullptr : ctx->d_upair_pod; a.max_victims = max_victims;
    pre_budgets(ctx, a, budgets);
    Prof prof(ctx);
    launch_uns_prep(ctx, d_pod_off, d_cand_off, n_pod, n_claim, n_pair);
    if ((rc = launch_running_lists(ctx, a, prof, false))) return rc;
    if ((rc = launch_preempt_pairs(ctx, a, s))) return rc;
    k_spre_reduce<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, st>>>(a, s);
    ctx->launches += 1;
    if (max_victims && hi > lo) {
        // in words from pod 0's partial: the best EVICT position at 1, the row from 8 (unit 2); 4 * stride words per pod
        uint32_t* part = reinterpret_cast<uint32_t*>(s.part + 1);
        launch_preempt_victims(ctx, a, part + 1, 4 * s.stride, part + 8, 4 * s.stride);
    }
    prof.mark();
    PreMerge m; memset(&m, 0, sizeof m);
    m.part = s.part; m.pairs = s.pairs; m.stride = s.stride;
    m.claims = a.claims; m.pod_off = d_pod_off; m.n_pod = n_pod;
    m.cand_nodes = a.cand_nodes; m.cand_off = a.cand_off; m.n_pair = n_pair; m.n_node = ctx->n_node;
    m.sel = a.sel; m.max_victims = max_victims; m.gate = a.gate;
    merge_bounds(ctx, gather, m.bounds);
    m.pair_status = d_pair_status; m.pair_victims = d_pair_victims;
    m.pod_node = d_pod_node; m.pod_status = d_pod_status; m.n_victims = d_n_victims; m.victims = max_victims ? d_victims : nullptr;
    m.pair_viol = d_pair_violations; m.pod_viol = d_pod_violations;
    const uint32_t n4 = (uint32_t)(1 + (size_t)n_pod * s.stride + (want_pairs ? ((size_t)n_pair + 1) / 2 : 0));
    const PeerExchange x = push_slice(ctx, ctx->pre_x, gather, s.part, n4);
    if (gather) m.slice4 = (uint32_t)(ctx->pre_x.slice / 16);
    const size_t work = std::max(((size_t)n_pod + 7) / 8, want_pairs ? ((size_t)n_pair + 255) / 256 : 0);
    k_spre_merge<<<wait_grid(ctx, work), 256, 0, st>>>(x, m);
    ctx->launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded preemption launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int dra_preempt_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                    const uint32_t* d_pod_off, const int32_t* d_prio, uint32_t n_pod,
                                    const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                    const dra_running_pods* running,
                                    uint8_t* d_pair_status, uint32_t* d_pair_victims,
                                    uint32_t* d_pod_node, uint8_t* d_pod_status, uint32_t* d_n_victims,
                                    uint32_t* d_victims, uint32_t max_victims, uint32_t flags) {
    return dra_preempt_pdb_batch_global_device(ctx, d_claims, n_claim, d_pod_off, d_prio, n_pod, d_cand_nodes, d_cand_off, n_pair,
                                               running, nullptr, d_pair_status, d_pair_victims, nullptr, d_pod_node,
                                               d_pod_status, d_n_victims, nullptr, d_victims, max_victims, flags);
}

int dra_set_shard_capacity(dra_ctx* ctx, uint32_t max_pairs) {
    if (!ctx) return DRA_E_INVAL;
    if (int rc = check_before_export(ctx, "dra_set_shard_capacity")) return rc;
    if (max_pairs > 0xFFFFFFF0u) return fail(ctx, DRA_E_INVAL, "dra_set_shard_capacity: max_pairs %u above 2^32 - 16", max_pairs);
    if (scap_units(max_pairs) > ((size_t)1 << 32) / 16)
        return fail(ctx, DRA_E_INVAL, "dra_set_shard_capacity: one rank's slice would exceed 4 GiB");
    ctx->shard_req.scap_pairs = max_pairs;
    return DRA_OK;
}

// Sharded pod capacity: offset checks and pair -> pod (k_uns_prep) -> the window's pairs into this rank's slice
// (k_pods_capacity) -> push to every peer -> wait + merge into the caller's buffers, with the per-pod sums (k_scap_merge).
// Enqueues only.
int dra_pod_capacity_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                         const uint32_t* d_pod_off, uint32_t n_pod,
                                         const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                         uint32_t max_copies, uint16_t* d_pair_copies, uint8_t* d_pair_stop,
                                         uint64_t* d_pod_total, uint32_t* d_pod_nodes, uint32_t flags) {
    if (!ctx || !d_pod_off || (n_claim && !d_claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_pod_capacity_batch_global_device: unknown flags 0x%x", flags);
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (max_copies < 1 || max_copies > 65535) return fail(ctx, DRA_E_INVAL, "max_copies %u outside [1, 65535]", max_copies);
    bool dense;
    if (int rc = check_dev_cands(ctx, d_cand_nodes, d_cand_off, n_pod, n_pair, true, dense)) return rc;
    if (n_pod > (1u << 26)) return fail(ctx, DRA_E_INVAL, "n_pod %u too large for the sharded call (2^26)", n_pod);
    const bool gather = ctx->world > 1;
    const uint32_t max_pairs = ctx->shard_rsv.scap_pairs;
    // no exchange reserved: even a call with no pairs pushes a header and raises flags, which would land in the peers'
    // buffers at offset 0
    if (int rc = check_world(ctx, "the merge needs", true, [&] {
            if (max_pairs) return (int)DRA_OK;
            return fail(ctx, DRA_E_STATE, "world > 1: dra_set_shard_capacity(max_pairs > 0) was not called before dra_shard_export");
        }, -1, [&] {
            if (n_pair <= max_pairs) return (int)DRA_OK;
            return fail(ctx, DRA_E_INVAL, "n_pair %u exceeds the max_pairs (%u) of dra_set_shard_capacity before dra_shard_export", n_pair, max_pairs);
        }))
        return rc;
    if (n_pair && !d_pair_copies) return fail(ctx, DRA_E_INVAL, "pair_copies is NULL");
    ctx->chain = DRA_K_POD_CAPACITY_SHARD; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;                         // every rank sees the same n_pod: none of them exchanges anything
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    // world > 1: peer_setup sized both for max_pairs, so these never reallocate there
    if ((rc = grow(ctx, ctx->d_scap_part, ctx->cap_scap_part, scap_units(n_pair)))) return rc;
    if (!dense && (rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, n_pair))) return rc;
    cudaStream_t st = ctx->stream;
    const uint32_t lo = gather ? ctx->shard_lo : 0u, hi = gather ? ctx->shard_hi : ctx->n_node;   // world 1: every node
    const uint32_t* gate = ctx->d_err + ERR_BAD_OFFSETS;
    CapArgs a; memset(&a, 0, sizeof a);
    a.claims = (const uint4*)d_claims; a.pod_off = d_pod_off; a.n_pod = n_pod;
    a.cand_nodes = dense ? nullptr : d_cand_nodes; a.cand_off = dense ? nullptr : d_cand_off;
    a.pair_pod = dense ? nullptr : ctx->d_upair_pod; a.n_pair = n_pair;
    a.inv = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.tbl = ctx->d_tbl; a.sel = sel_of(ctx);
    a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u; a.max_copies = max_copies;
    a.node_lo = lo; a.n_win = hi - lo; a.n_walk = dense ? n_pod * a.n_win : n_pair;   // (n_pod * n_win <= n_pair)
    uint4* part = ctx->d_scap_part;
    const size_t copies4 = ((size_t)a.n_walk + 7) / 8, stops4 = d_pair_stop ? ((size_t)a.n_walk + 15) / 16 : 0;
    a.pair_copies = reinterpret_cast<uint16_t*>(part + 1);
    a.pair_stop = d_pair_stop ? reinterpret_cast<uint8_t*>(part + 1 + copies4) : nullptr;
    a.gate = gate;
    Prof prof(ctx);
    launch_uns_prep(ctx, d_pod_off, d_cand_off, n_pod, n_claim, n_pair);
    if ((rc = launch_capacity(ctx, a))) return rc;
    prof.mark();
    CapMerge m; memset(&m, 0, sizeof m);
    m.part = part; m.cand_nodes = a.cand_nodes; m.cand_off = a.cand_off;
    m.n_pod = n_pod; m.n_pair = n_pair; m.n_node = ctx->n_node;
    merge_bounds(ctx, gather, m.bounds);
    m.gate = gate;
    m.pair_copies = d_pair_copies; m.pair_stop = d_pair_stop; m.pod_total = (unsigned long long*)d_pod_total; m.pod_nodes = d_pod_nodes;
    if (gather) {
        m.slice4 = (uint32_t)(ctx->scap_x.slice / 16);
        CU(cudaMemcpyAsync(part, gate, 4, cudaMemcpyDeviceToDevice, st));   // the header: this rank's fault word
    }
    const PeerExchange x = push_slice(ctx, ctx->scap_x, gather, part, (uint32_t)(1 + copies4 + stops4));
    k_scap_merge<<<wait_grid(ctx, (n_pod + 7) / 8), 256, 0, st>>>(x, m);
    ctx->launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded pod capacity launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int dra_set_shard_why(dra_ctx* ctx, uint32_t max_pairs) {
    if (!ctx) return DRA_E_INVAL;
    if (int rc = check_before_export(ctx, "dra_set_shard_why")) return rc;
    if (max_pairs > 0xFFFFFFF0u) return fail(ctx, DRA_E_INVAL, "dra_set_shard_why: max_pairs %u above 2^32 - 16", max_pairs);
    if (swhy_units(max_pairs) > ((size_t)1 << 32) / 16)
        return fail(ctx, DRA_E_INVAL, "dra_set_shard_why: one rank's slice would exceed 4 GiB");
    ctx->shard_req.swhy_pairs = max_pairs;
    return DRA_OK;
}

// Sharded reasons of UnsuitableNodes: offset checks and pair -> pod (k_uns_prep) -> the window's reasons into this rank's
// slice (k_unsuitable<..., WIN, WHY>) -> push to every peer -> wait + merge into the caller's buffers, with the tallies
// (k_swhy_merge).  Enqueues only.
int dra_unsuitable_why_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                           const uint32_t* d_pod_off, uint32_t n_pod,
                                           const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                           uint8_t* d_pair_why, uint32_t* d_pair_claim,
                                           uint32_t* d_pod_why, uint32_t* d_claim_blocks, uint32_t flags) {
    if (!ctx || !d_pod_off || (n_claim && !d_claims)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE) return fail(ctx, DRA_E_INVAL, "dra_unsuitable_why_batch_global_device: unknown flags 0x%x", flags);
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    bool dense;
    if (int rc = check_dev_cands(ctx, d_cand_nodes, d_cand_off, n_pod, n_pair, true, dense)) return rc;
    if (n_pod > (1u << 26)) return fail(ctx, DRA_E_INVAL, "n_pod %u too large for the sharded call (2^26)", n_pod);
    const bool gather = ctx->world > 1;
    if (int rc = check_world(ctx, "the merge needs", true, [ctx] { return swhy_reserved(ctx); }, -1,
                             [&] { return swhy_fits(ctx, n_pair); }))
        return rc;
    const WhyOut w{d_pair_why, d_pair_claim, d_pod_why, d_claim_blocks};
    if (int rc = why_check(ctx, &w, n_pair)) return rc;
    ctx->chain = DRA_K_UNSUITABLE_WHY_SHARD; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;                         // every rank sees the same n_pod: none of them exchanges anything
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    const uint32_t lo = gather ? ctx->shard_lo : 0u, hi = gather ? ctx->shard_hi : ctx->n_node;   // world 1: every node
    const uint32_t n_walk = dense ? n_pod * (hi - lo) : n_pair;                                 // (n_pod * n_win <= n_pair)
    // (world > 1: peer_setup sized d_upair_pod for max_pairs too, so it never reallocates there)
    if ((rc = swhy_buffers(ctx, w, n_walk, n_claim)) ||
        (!dense && (rc = grow(ctx, ctx->d_upair_pod, ctx->cap_upair_pod, n_pair)))) return rc;
    const uint32_t* gate = ctx->d_err + ERR_BAD_OFFSETS;
    UnsArgs a; memset(&a, 0, sizeof a);
    a.claims = (const uint4*)d_claims; a.pod_off = d_pod_off; a.n_pod = n_pod;
    a.cand_nodes = dense ? nullptr : d_cand_nodes; a.cand_off = dense ? nullptr : d_cand_off;
    a.pair_pod = dense ? nullptr : ctx->d_upair_pod;
    a.inv = ctx->d_inv_live; a.node_off = ctx->d_node_off; a.n_node = ctx->n_node; a.tbl = ctx->d_tbl; a.sel = sel_of(ctx);
    a.exhaustive = (flags & DRA_F_EXHAUSTIVE) ? 1u : 0u;
    a.node_lo = lo; a.n_win = hi - lo; a.n_walk = n_walk;
    a.gate = gate;
    swhy_slice(ctx, n_walk, a.why, a.why_claim);
    Prof prof(ctx);
    launch_uns_prep(ctx, d_pod_off, d_cand_off, n_pod, n_claim, n_pair);
    if (n_walk && (rc = launch_unsuitable(ctx, a, true, true))) return rc;
    prof.mark();
    if ((rc = launch_swhy_merge(ctx, w, gate, n_walk, a.cand_nodes, a.cand_off, n_pod, n_pair, n_claim))) return rc;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded unsuitable reasons launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int dra_set_shard_preempt_place(dra_ctx* ctx, uint32_t max_pods, uint32_t max_pairs, uint32_t max_run) {
    if (!ctx) return DRA_E_INVAL;
    if (int rc = check_before_export(ctx, "dra_set_shard_preempt_place")) return rc;
    if (max_pods > (1u << 26) || max_pairs > 0xFFFFFFF0u || max_run > (1u << 26))
        return fail(ctx, DRA_E_INVAL, "dra_set_shard_preempt_place: sizes too large (max_pods, max_run <= 2^26, max_pairs <= 2^32 - 16)");
    ShardSizes& z = ctx->shard_req;
    z.spp_pods = max_pods; z.spp_pairs = max_pairs; z.spp_run = max_run;
    return DRA_OK;
}

// Sharded preempt and place: the world's state into the scratch inventory (own range from the live copy, the others over
// the inventory sync's exchange: k_peer_push, k_isync_copy) -> §15's chain on the scratch copy, identical on every rank
// (k_pre_running, the counting sort, k_pre_vsort, k_spp_prep, the counting sort of the pairs, k_pods_preempt_place) ->
// the caller's outputs and the own GPU range back into the live copy (k_spp_final).  Enqueues only.
int dra_preempt_place_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                          const uint32_t* d_pod_off, const int32_t* d_prio, uint32_t n_pod,
                                          const uint32_t* d_cand_nodes, const uint32_t* d_cand_off, uint32_t n_pair,
                                          const dra_running_pods* running, const uint32_t* d_out_off, uint32_t n_out,
                                          uint32_t* d_pod_node, uint8_t* d_pod_status, uint32_t* d_evicted_by, uint32_t flags) {
    if (!ctx || !d_pod_off || !running || !running->pod_off || (n_claim && !d_claims) ||
        (n_pod && (!d_prio || !d_pod_node || !d_pod_status)))
        return DRA_E_INVAL;
    const dra_running_pods& R = *running;
    if ((R.n_claim && !R.claims) || (R.n_pod && (!R.prio || !d_evicted_by)) || (R.n_out && !R.out)) return DRA_E_INVAL;
    QUIESCE();
    if (flags & ~DRA_F_EXHAUSTIVE)
        return fail(ctx, DRA_E_INVAL, "dra_preempt_place_batch_global_device: unknown flags 0x%x (DRA_F_FRESH_INVENTORY is not taken)", flags);
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (n_pod > (1u << 26) || R.n_pod > (1u << 26)) return fail(ctx, DRA_E_INVAL, "batch too large for the sharded call (2^26)");
    if (int rc = check_slots(ctx, n_claim, n_out, d_out_off != nullptr)) return rc;
    if (!n_pod && n_claim) return fail(ctx, DRA_E_INVAL, "pod_off must span [0, n_claim]: no pods for %u claims", n_claim);
    bool dense;
    if (int rc = check_dev_cands(ctx, d_cand_nodes, d_cand_off, n_pod, n_pair, false, dense)) return rc;
    if (ctx->n_node > PL_POS) return fail(ctx, DRA_E_INVAL, "more than %u nodes", PL_POS);
    const uint64_t walk64 = dense ? (uint64_t)n_pod * ctx->n_node : n_pair;     // the pairs the walk judges
    if (walk64 > 0xFFFFFFF0u) return fail(ctx, DRA_E_INVAL, "too many (pod, node) pairs");
    const uint32_t walk = (uint32_t)walk64;
    const bool gather = ctx->world > 1;
    const ShardSizes& z = ctx->shard_rsv;
    if (int rc = check_world(ctx, "the exchange needs", true, [&] {
            if (int rc = check_inv_exchange(ctx)) return rc;
            if (z.spp_pods) return (int)DRA_OK;
            return fail(ctx, DRA_E_STATE, "dra_set_shard_preempt_place was not called before dra_shard_export");
        }, n_out, [&] {
            if (n_pod <= z.spp_pods && walk <= z.spp_pairs && R.n_pod <= z.spp_run) return (int)DRA_OK;
            return fail(ctx, DRA_E_INVAL, "n_pod %u / pairs %u / running pods %u exceed the sizes of dra_set_shard_preempt_place before "
                        "dra_shard_export (%u / %u / %u)", n_pod, walk, R.n_pod, z.spp_pods, z.spp_pairs, z.spp_run);
        }))
        return rc;
    ctx->chain = DRA_K_PREEMPT_PLACE_SHARD; ctx->chain_tile = 0;
    if (!n_pod) return DRA_OK;                         // every rank sees the same n_pod: none of them exchanges anything
    CallScope scope{ctx};
    int rc = scope.open(gather);
    if (rc) return rc;
    if ((rc = spp_buffers(ctx, n_pod, walk, R.n_pod))) return rc;
    if (ctx->pp_occ < 0 && (rc = preload_preempt_place_shard(ctx))) return rc;
    if (ctx->pp_occ < 1) return fail(ctx, DRA_E_CUDA, "k_pods_preempt_place: no CTA can be resident");
    // The table is this context's own: every rank computes the whole of it, so no packet moves and the gather's epochs,
    // parities and cursors are left to the calls that gather
    if ((rc = grow_set(ctx, ctx->cap_gtable, (size_t)n_out + 16, ctx->d_gtable))) return rc;
    uint2* table = ctx->d_gtable;
    cudaStream_t st = ctx->stream;
    const Err err = err_of(ctx);
    // world 1: the rank owns every GPU
    const uint32_t gpu_lo = gather ? ctx->h_node_off[ctx->shard_bounds[ctx->rank]] : 0u;
    const uint32_t gpu_hi = gather ? ctx->h_node_off[ctx->shard_bounds[ctx->rank + 1]] : ctx->n_gpu;
    Prof prof(ctx);
    CU(cudaMemsetAsync(ctx->d_spp_gate, 0, 4, st));
    CU(cudaMemcpyAsync(ctx->d_spp_inv, ctx->d_inv_live, (size_t)ctx->n_gpu * 16, cudaMemcpyDeviceToDevice, st));
    if (gather) {
        const PeerExchange x = bind_exchange(ctx, ctx->isync_x);
        InvSync s; memset(&s, 0, sizeof s);
        s.inv = ctx->d_spp_inv; s.n_gpu = ctx->n_gpu; s.own_lo = gpu_lo; s.own_hi = gpu_hi;
        s.elect = (uint32_t*)(ctx->peer_local + ctx->isync_x.flags) + PEER_MAX;
        k_peer_push<<<push_grid(ctx, gpu_hi - gpu_lo), 256, 0, st>>>(x, ctx->d_inv_live, gpu_lo, gpu_hi);
        k_isync_copy<<<wait_grid(ctx, (ctx->n_gpu + 255) / 256), 256, 0, st>>>(x, s);
        // one verdict for the world: the call fails on every rank or on none
        k_spp_agree<<<1, 32, 0, st>>>(bind_exchange(ctx, ctx->spp_x), s.elect, x.seq, ctx->d_spp_gate);
        ctx->launches += 3;
    }
    if (n_out) CU(cudaMemsetAsync(table, 0, (size_t)n_out * 8, st));
    CU(cudaMemsetAsync(ctx->d_place_cursor, 0, ((size_t)ctx->n_node + 1) * 4, st));
    CU(cudaMemsetAsync(ctx->d_pp_judged, 0, ((size_t)ctx->n_node + 1) * 4, st));
    if (R.n_pod) CU(cudaMemsetAsync(ctx->d_pp_evicted, 0xFF, (size_t)R.n_pod * 4, st));

    PreArgs a = pre_args(ctx, (const uint4*)d_claims, d_pod_off, d_prio, n_pod, dense ? nullptr : d_cand_nodes,
                         dense ? nullptr : d_cand_off, walk, R, ctx->d_spp_inv, flags);
    // the running lists (§14), on global GPU indices: every rank finds the same faults
    if ((rc = launch_running_lists(ctx, a, prof, true))) return rc;
    // the checks of the pending arrays and the visit lists (§13)
    PlaceArgs pl; memset(&pl, 0, sizeof pl);
    pl.claims = a.claims; pl.pod_off = d_pod_off; pl.n_pod = n_pod;
    pl.cand_nodes = a.cand_nodes; pl.cand_off = a.cand_off;
    pl.out_off = d_out_off; pl.out = table;
    pl.state = ctx->d_place_state; pl.pairs = ctx->d_podrec;
    pl.sorted = ctx->d_sorted; pl.list_off = ctx->d_claim_off; pl.cursor = ctx->d_place_cursor;
    pl.inv_src = ctx->d_spp_inv; pl.inv_dst = ctx->d_spp_inv; pl.node_off = ctx->d_node_off; pl.tbl = ctx->d_tbl;
    pl.n_node = ctx->n_node; pl.exhaustive = a.exhaustive; pl.sel = a.sel; pl.err = err;
    PpArgs pp{ctx->d_pp_pending, ctx->d_pp_evicted, ctx->d_pp_judged};
    SppArgs s; memset(&s, 0, sizeof s);
    s.n_claim = n_claim; s.n_pair = n_pair; s.n_out = n_out; s.gate = ctx->d_spp_gate; s.err_dev = ctx->d_err;
    s.pod_node_src = ctx->d_pre_node; s.pod_status_src = ctx->d_pre_pst; s.evicted_src = ctx->d_pp_evicted;
    s.pod_node = d_pod_node; s.pod_status = d_pod_status; s.evicted_by = d_evicted_by; s.n_pod = n_pod; s.rn_pod = R.n_pod;
    s.inv_src = ctx->d_spp_inv; s.inv_dst = ctx->d_inv_live; s.gpu_lo = gpu_lo; s.gpu_hi = gpu_hi;
    k_spp_prep<<<(unsigned)(((size_t)n_pod * 32 + 255) / 256), 256, 0, st>>>(a, pl, pp, s);
    ctx->launches += 1;
    // A candidate form with no pair sorts nothing, so the visit lists are zeroed instead: the walk must not read the
    // offsets an earlier call's sort left in d_claim_off (an Allocate's claims by node), as lists of this call's pairs
    if (!dense && !n_pair) CU(cudaMemsetAsync(ctx->d_claim_off, 0, ((size_t)ctx->n_node + 2) * 4, st));
    if (!dense && n_pair &&
        (rc = launch_sort(ctx, ctx->d_podrec, n_pair, nullptr, nullptr, 0, 0, prof, ctx->d_spp_inv, LA_NONE, ctx->n_node, ctx->d_node_off)))
        return rc;
    if (ctx->n_node) {                 // every CTA resident (shard_walk_grid); the walk itself waits for no peer
        PreArgs aw = a;
        aw.gate = ctx->d_spp_gate;
        k_pods_preempt_place<4><<<shard_walk_grid(ctx, ctx->pp_occ, gather, ctx->n_node), 128, 0, st>>>(aw, pl, pp);
        ctx->launches += 1;
    }
    const uint32_t fin = std::max(std::max(n_pod, R.n_pod), gpu_hi - gpu_lo);
    k_spp_final<<<std::max(1u, std::min((fin + 255) / 256, (uint32_t)ctx->n_sm * 2u)), 256, 0, st>>>(s);
    ctx->launches += 1;
    ctx->chain |= DRA_K_PREEMPT_PLACE_SHARD;
    prof.mark();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded preempt-and-place launch: %s", cudaGetErrorString(e));
    ctx->gather_table = (const dra_out_rec*)table; ctx->gather_n_per = n_out; ctx->gather_len = n_out;
    return DRA_OK;
}

// Inventory sync: this rank's GPU range into every peer's staging (k_peer_push) -> flags, wait, and the copy of every other
// rank's range into the live copy (k_isync_copy).  Enqueues only.
int dra_shard_sync_inventory_device(dra_ctx* ctx) {
    if (!ctx) return DRA_E_INVAL;
    QUIESCE();
    if (ctx->world <= 1) return DRA_OK;
    if (int rc = check_world(ctx, "the sync needs", true, [ctx] { return check_inv_exchange(ctx); }, -1, no_check)) return rc;
    CU(cudaSetDevice(ctx->device));
    const PeerExchange x = bind_exchange(ctx, ctx->isync_x);
    InvSync s; memset(&s, 0, sizeof s);
    s.inv = ctx->d_inv_live; s.n_gpu = ctx->n_gpu;
    s.elect = (uint32_t*)(ctx->peer_local + ctx->isync_x.flags) + PEER_MAX;
    s.own_lo = ctx->h_node_off[ctx->shard_bounds[ctx->rank]]; s.own_hi = ctx->h_node_off[ctx->shard_bounds[ctx->rank + 1]];
    k_peer_push<<<push_grid(ctx, s.own_hi - s.own_lo), 256, 0, ctx->stream>>>(x, s.inv, s.own_lo, s.own_hi);
    k_isync_copy<<<wait_grid(ctx, (ctx->n_gpu + 255) / 256), 256, 0, ctx->stream>>>(x, s);
    ctx->launches += 2;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "inventory sync launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

// Sharded Deallocate: the slot-range check over every claim (k_dealloc_check) -> the gated apply on this rank's GPU range
// (k_dealloc, a programmatic dependent of the check).  Spec §9 updates commute and touch only the GPU a record names, so no
// rank exchanges anything and none waits for a peer.  Enqueues only; allocates nothing.
int dra_deallocate_batch_global_device(dra_ctx* ctx, const dra_claim_rec* d_claims, uint32_t n_claim,
                                       const uint32_t* d_out_off, const dra_out_rec* d_out, uint32_t n_out) {
    if (!ctx || (n_claim && (!d_claims || !d_out))) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (!ctx->shard_on) return fail(ctx, DRA_E_STATE, "dra_set_shard has not been called");
    if (ctx->shard_hi > ctx->n_node) return fail(ctx, DRA_E_STATE, "the shard [%u, %u) lies outside the inventory's %u nodes", ctx->shard_lo, ctx->shard_hi, ctx->n_node);
    if (int rc = check_slots(ctx, n_claim, n_out, d_out_off != nullptr)) return rc;
    if (!n_claim) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    const Err err = err_of(ctx);
    const uint32_t gpu_lo = ctx->h_node_off[ctx->shard_lo], gpu_hi = ctx->h_node_off[ctx->shard_hi];
    k_dealloc_check<<<std::max(1u, std::min((n_claim + 255) / 256, (uint32_t)ctx->n_sm * 4u)), 256, 0, ctx->stream>>>(
        (const uint4*)d_claims, n_claim, d_out_off, n_out, ctx->n_node, err);
    CU(launch_k(k_dealloc, dim3((n_claim + 255) / 256), dim3(256), 0, ctx->stream, pdl_attr(ctx),
                (const uint4*)d_claims, n_claim, d_out_off, (const uint2*)d_out, n_out, (uint32_t*)ctx->d_inv_live, gpu_lo, gpu_hi,
                ctx->n_node, (const uint32_t*)(ctx->d_err + ERR_BAD_DEALLOC), err));
    ctx->launches += 2;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "sharded Deallocate launch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int dra_gather_table(dra_ctx* ctx, const dra_out_rec** d_table, uint32_t* n_per_rank) {
    if (!ctx || !d_table) return DRA_E_INVAL;
    if (!ctx->gather_table) return fail(ctx, DRA_E_STATE, "no gather has run");
    *d_table = ctx->gather_table;
    if (n_per_rank) *n_per_rank = ctx->gather_n_per;
    return DRA_OK;
}

int dra_gather_read(dra_ctx* ctx, dra_out_rec* out_all, uint32_t n_rec) {
    if (!ctx || !out_all) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->gather_table) return fail(ctx, DRA_E_STATE, "no gather has run");
    if (n_rec > (ctx->gather_len ? ctx->gather_len : (uint32_t)ctx->world * ctx->gather_n_per)) return fail(ctx, DRA_E_INVAL, "n_rec %u exceeds the table", n_rec);
    CU(cudaSetDevice(ctx->device));
    const size_t rb = (size_t)n_rec * 8;
    const bool direct = is_pinned(out_all, rb);
    int rc;
    if (!direct && (rc = grow_pinned(ctx, ctx->h_out, ctx->h_out_cap, rb))) return rc;
    CU(cudaMemcpyAsync(direct ? (void*)out_all : (void*)ctx->h_out, ctx->gather_table, rb, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if ((rc = check_err(ctx))) return rc;
    if (!direct) memcpy(out_all, ctx->h_out, rb);
    return DRA_OK;
}

// ---- adjacent integer searches, batched (SURVEY §8f-4) ------------------------------------------------
int dra_mps_limits_batch(dra_ctx* ctx, const int64_t* bytes, uint32_t n, int64_t* mib, uint8_t* valid) {
    if (!ctx || (n && (!bytes || !mib || !valid))) return DRA_E_INVAL;
    QUIESCE();
    if (!n) return DRA_OK;
    CU(cudaSetDevice(ctx->device));
    void *d_b = nullptr, *d_m = nullptr, *d_v = nullptr;
    CU(cudaMalloc(&d_b, (size_t)n * 8)); CU(cudaMalloc(&d_m, (size_t)n * 8)); CU(cudaMalloc(&d_v, n));
    cudaError_t e = cudaMemcpyAsync(d_b, bytes, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream);
    k_mps_limits<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const long long*)d_b, n, (long long*)d_m, (uint8_t*)d_v);
    ctx->launches += 1;
    if (e == cudaSuccess) e = cudaMemcpyAsync(mib, d_m, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(valid, d_v, n, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d_b); cudaFree(d_m); cudaFree(d_v);
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "dra_mps_limits_batch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

int dra_imex_offsets_batch(dra_ctx* ctx, const int32_t* used, const uint32_t* dom_off, uint32_t n_dom, int32_t step, int32_t limit, int32_t* out) {
    if (!ctx || !dom_off || (n_dom && !out) || step <= 0 || limit < 0) return DRA_E_INVAL;
    QUIESCE();
    if (!n_dom) return DRA_OK;
    const uint32_t n_used = dom_off[n_dom];
    if (n_used && !used) return DRA_E_INVAL;
    CU(cudaSetDevice(ctx->device));
    void *d_u = nullptr, *d_o = nullptr, *d_r = nullptr;
    CU(cudaMalloc(&d_u, (size_t)n_used * 4 + 16)); CU(cudaMalloc(&d_o, ((size_t)n_dom + 1) * 4)); CU(cudaMalloc(&d_r, (size_t)n_dom * 4));
    cudaError_t e = cudaSuccess;
    if (n_used) e = cudaMemcpyAsync(d_u, used, (size_t)n_used * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_o, dom_off, ((size_t)n_dom + 1) * 4, cudaMemcpyHostToDevice, ctx->stream);
    k_imex_offsets<<<(n_dom + 7) / 8, 256, 0, ctx->stream>>>((const int*)d_u, (const uint32_t*)d_o, n_dom, step, limit, (int*)d_r);
    ctx->launches += 1;
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_r, (size_t)n_dom * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d_u); cudaFree(d_o); cudaFree(d_r);
    if (e != cudaSuccess) return fail(ctx, DRA_E_CUDA, "dra_imex_offsets_batch: %s", cudaGetErrorString(e));
    return DRA_OK;
}

// One-time calibration of the single-launch / sort-path crossover on THIS device and THIS inventory: synthetic MIG claims
// (uniform over the nodes) at a few batch sizes through both chains, CUDA events, best of 5; the live inventory is
// saved and restored.  Sets the claim count up to which dra_allocate_batch takes the single-launch kernel.
int dra_calibrate(dra_ctx* ctx, uint32_t* crossover_claims) {
    if (!ctx) return DRA_E_INVAL;
    QUIESCE();
    if (!ctx->d_inv_live || !ctx->n_node) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    CU(cudaSetDevice(ctx->device));
    const uint32_t sizes[] = {2000, 4000, 6000, 8000, 10000, 12000, 14000, 16000, 20000, 24000};
    const uint32_t n_max = 24000;
    int rc = ensure_batch(ctx, n_max, n_max, true);
    if (rc) return rc;
    std::vector<dra_claim_rec> h(n_max);
    uint64_t x = 0x9E3779B97F4A7C15ull;
    for (uint32_t i = 0; i < n_max; ++i) {
        x ^= x << 13; x ^= x >> 7; x ^= x << 17;
        h[i].kind = DRA_KIND_MIG; h[i].profile = (uint8_t)((x >> 40) % 3); h[i].count = 1;
        h[i].node = (uint32_t)(x % ctx->n_node); h[i].mem_limit_mib = 0; h[i].group = 0;
    }
    uint4* d_save = nullptr;
    CU(cudaMalloc((void**)&d_save, (size_t)ctx->n_gpu * 16 + 16));
    CU(cudaMemcpy(d_save, ctx->d_inv_live, (size_t)ctx->n_gpu * 16, cudaMemcpyDeviceToDevice));
    CU(cudaMemcpy(ctx->d_claims, h.data(), (size_t)n_max * 16, cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1; CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
    const uint32_t saved_flags = ctx->cfg_flags;
    const uint32_t saved_a = ctx->fused_max_one_wave, saved_b = ctx->fused_max_multi;
    const bool prof = ctx->profiling; ctx->profiling = false;
    const uint32_t saved_chain = ctx->chain, saved_tile = ctx->chain_tile;   // (calibration runs are no Allocate call)
    uint32_t best = 0; bool lost = false;
    for (uint32_t n : sizes) {
        float t[2] = {1e30f, 1e30f};
        for (int path = 0; path < 2 && rc == DRA_OK; ++path) {
            ctx->cfg_flags = (saved_flags & ~DRA_CFG_NO_FUSED) | (path ? DRA_CFG_NO_FUSED : 0u);
            ctx->fused_max_one_wave = ctx->fused_max_multi = path ? 0u : 0xFFFFFFFFu;
            if (path == 0 && !fused_plan(ctx, n, DRA_F_FRESH_INVENTORY, ctx->n_node).fused) { t[0] = 1e30f; continue; }   // not launchable at this size
            for (int rep = 0; rep < 6 && rc == DRA_OK; ++rep) {
                cudaEventRecord(e0, ctx->stream);
                rc = launch_allocate(ctx, ctx->d_claims, n, nullptr, ctx->d_out, n, DRA_F_FRESH_INVENTORY);
                cudaEventRecord(e1, ctx->stream);
                if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = fail(ctx, DRA_E_CUDA, "calibration run failed");
                float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
                if (rep) t[path] = std::min(t[path], ms);
            }
        }
        if (rc) break;
        if (t[0] <= t[1] && !lost) best = n; else lost = true;          // the first size at which the sort path wins ends the range
    }
    ctx->cfg_flags = saved_flags; ctx->profiling = prof;
    ctx->chain = saved_chain; ctx->chain_tile = saved_tile;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaMemcpy(ctx->d_inv_live, d_save, (size_t)ctx->n_gpu * 16, cudaMemcpyDeviceToDevice);
    cudaFree(d_save);
    (void)check_err(ctx);
    if (rc) { ctx->fused_max_one_wave = saved_a; ctx->fused_max_multi = saved_b; return rc; }
    if ((int)(ctx->n_node + 1) <= ctx->n_sm) { ctx->fused_max_one_wave = best; ctx->fused_max_multi = saved_b; }
    else { ctx->fused_max_multi = best; ctx->fused_max_one_wave = saved_a; }
    ctx->state_epoch++;
    if (crossover_claims) *crossover_claims = best;
    return DRA_OK;
}

// ---- resident mode ---------------------------------------------------------------------------------------------------
int dra_serve_start(dra_ctx* ctx) {
    if (!ctx) return DRA_E_INVAL;
    if (!ctx->d_inv_live) return fail(ctx, DRA_E_STATE, "dra_set_inventory has not been called");
    if (!ctx->coop_ok || (int)(ctx->n_node + 1) > ctx->n_sm) return fail(ctx, DRA_E_STATE, "resident mode needs every node's CTA resident at once: %u nodes, %d SMs", ctx->n_node, ctx->n_sm);
    int rc = serve_stop(ctx);
    if (rc) return rc;
    return serve_start(ctx);
}
int dra_serve_stop(dra_ctx* ctx) { if (!ctx) return DRA_E_INVAL; return serve_stop(ctx); }
uint64_t dra_serve_batches(const dra_ctx* ctx) { return ctx ? ctx->serve_batches : 0; }

// ---- host memory + instrumentation -----------------------------------------------------------------

void* dra_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    std::lock_guard<std::mutex> lk(g_pin_mu);
    g_pinned[(uintptr_t)p] = bytes ? bytes : 16;
    return p;
}

void dra_host_free(void* p) {
    if (!p) return;
    { std::lock_guard<std::mutex> lk(g_pin_mu); g_pinned.erase((uintptr_t)p); }
    cudaFreeHost(p);
}

uint64_t dra_launch_count(const dra_ctx* ctx) { return ctx ? ctx->launches : 0; }

int dra_debug_last_chain(const dra_ctx* ctx, uint32_t* kernels, uint32_t* hist_tile) {
    if (!ctx) return DRA_E_INVAL;
    if (kernels) *kernels = ctx->chain;
    if (hist_tile) *hist_tile = ctx->chain_tile;
    return DRA_OK;
}

namespace { __global__ void k_noop(int x) { extern __shared__ uint8_t sm[]; if (x == 12345) sm[0] = 1; } }

// Instrumentation: enqueue an empty kernel with the given shape (calibrates the launch floor of the box).
int dra_debug_noop(dra_ctx* ctx, uint32_t grid, uint32_t block, uint32_t smem) {
    if (!ctx) return DRA_E_INVAL;
    QUIESCE();
    CU(cudaSetDevice(ctx->device));
    if (smem > 48 * 1024) CU(cudaFuncSetAttribute(k_noop, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_noop<<<grid, block, smem, ctx->stream>>>(0);
    return DRA_OK;
}

int dra_debug_serve_times(dra_ctx* ctx, unsigned long long* four) {
    if (!ctx || !four || !ctx->d_go) return 0;
    cudaSetDevice(ctx->device);
    if (serve_stop(ctx)) return 0;
    cudaMemcpy(four, ctx->d_go + 32, 32, cudaMemcpyDeviceToHost);
    return 4;
}

int dra_debug_shard_times(dra_ctx* ctx, unsigned long long* two) {
    if (!ctx || !two || !ctx->d_sc_times) return 0;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaMemcpy(two, ctx->d_sc_times, 16, cudaMemcpyDeviceToHost);
    return 2;
}

int dra_debug_timeline(dra_ctx* ctx, unsigned long long* host, uint32_t n) {
    if (!ctx || !host || !ctx->d_timeline) return 0;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    uint32_t m = std::min(n, ctx->tl_n);
    cudaMemcpy(host, ctx->d_timeline, (size_t)m * 8, cudaMemcpyDeviceToHost);
    return (int)m;
}

int dra_set_profiling(dra_ctx* ctx, int enabled) {
    if (!ctx) return DRA_E_INVAL;
    ctx->profiling = enabled != 0;
    return DRA_OK;
}

int dra_get_timings(dra_ctx* ctx, float* us, int n) {
    if (!ctx || !us) return 0;
    int m = std::min(n, 5);
    for (int i = 0; i < m; ++i) us[i] = ctx->timings[i];
    return m;
}

}  // extern "C"
