// dra_device.cuh — sm_90a kernels of the allocation hot path (spec/ALLOCATION.md).
//
// Pipeline of one Allocate batch (all integer / bitwise, HBM-bound, no tensor cores):
//   k_bucket_hist    stable counting sort, pass 1: per-tile node histogram + stable intra-tile rank
//                    (__match_any_sync gives every lane its rank among equal-node lanes)
//   k_bucket_scan    pass 2: per-node exclusive scan over tiles, node offsets (CSR claim_off)
//   k_bucket_scatter pass 3: claims -> node-sorted array, first OutRec slot embedded in the record
//   k_pack           one warp per node, one lane per GPU: the node's GpuRecs and its claim span are
//                    staged into shared memory with 1-D TMA bulk copies (cp.async.bulk + mbarrier), each
//                    claim is tested on all GPUs at once, __ballot_sync + __ffs pick lowest GPU / lowest
//                    start (first-fit), the winner lane updates its register-resident occupancy mask.
//   k_unsuitable     one warp per (pod, candidate node) pair, same step function on a snapshot
//   k_pods_place     place pods (spec §13): persistent, a warp walks each of its nodes' visit lists with a cursor;
//                    sharded (<4, true>): the rank's node window, pod states replicated on every rank (k_splace_*)
//   k_pods_preempt   preemption (spec §14): per (pod, candidate) pair, W lanes, the victims by remove-all-then-reprieve;
//                    sharded: the same kernel on the rank's node window, per-pod partials merged on every rank (k_spre_*)
//   k_dealloc        inverse updates with atomics (sharded: behind k_dealloc_check, on the rank's GPU range only)
//
// What this replaces in the reference: the per-node search behind Allocate()/UnsuitableNodes() that
// north_star names (absent from the snapshot, SURVEY F1), over the device model of
// cmd/nvidia-dra-plugin/deviceinfo.go:30-64,199-204 and the placement enumeration of nvlib.go:244-295.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dra_alloc.h"

namespace dra {

constexpr uint32_t FULLMASK = 0xFFFFFFFFu;
constexpr uint32_t SEG = 32;          // claims per TMA segment
constexpr uint32_t RING = 4;          // ring slots per warp
constexpr uint32_t ERR_OUT_RANGE = 1u;    // index into the error-flag words
constexpr uint32_t ERR_NOT_SORTED = 2u;
constexpr uint32_t ERR_PEER_TIMEOUT = 3u;
constexpr uint32_t ERR_DEVICE_WAIT = 5u;     // a wait inside ONE GPU gave up (grid barrier, look-back): cannot happen unless CTAs were not co-scheduled
constexpr uint32_t ERR_SHARD_PLAN = 4u;      // sharded call: more claims fell into this shard than the launch was laid out for
constexpr uint32_t ERR_BAD_OFFSETS = 6u;     // sharded UnsuitableNodes: pod_off / cand_off not monotone or not spanning their arrays
constexpr uint32_t ERR_BAD_PODS = 7u;        // sharded pods Allocate: bad pod_off, slots outside n_out, or a rank's slots beyond its packet room
constexpr uint32_t ERR_BAD_DEALLOC = 8u;     // sharded Deallocate: a claim's slots outside n_out (nothing applied)
constexpr uint32_t ERR_WORDS = 9u;
constexpr uint32_t PEER_MAX = 16;         // ranks of one box

// Error flags: `dev` (device memory) gates later kernels of the same batch, `host` (mapped pinned
// memory) is what the host reads after the stream drains.  Idempotent plain stores, errors are rare.
struct Err {
    uint32_t* dev; volatile uint32_t* host;
    __device__ __forceinline__ void set(uint32_t which) const { dev[which] = 1u; host[which] = 1u; __threadfence_system(); }
};

// ---- record views ---------------------------------------------------------------------------------
// GpuRec   as uint4: x = busy | flags<<16 | model<<24 ; y = mem_free_mib ; z = node ; w = share|rsvd<<16
// ClaimRec as uint4: x = kind | profile<<8 | count<<16 ; y = node (sorted copy: first out slot) ;
//                    z = mem_limit_mib ; w = group
// OutRec   as uint2: x = gpu ; y = start | size<<8 | profile<<16 | status<<24

// Programmatic dependent launch (sort path: hist -> scan -> scatter -> pack).  A producer lets the next kernel's
// CTAs be scheduled early; a consumer blocks until the producer grid has completed and its writes are visible.
// Both are no-ops for a launch without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t addr = smem_u32(bar), ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    } while (!ok);
}
// 1-D TMA bulk copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void tma_prefetch_l2(const void* g, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(g), "r"(bytes) : "memory");
}

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m;
}


// Lanes whose key equals mine, as a mask — __match_any_sync semantics built from one ballot per key bit.
// MATCH.ANY serialises over the distinct values in the warp (~29 of 32 for node keys) on a unit shared by
// the SM; log2(n_node) VOTEs pipeline.  Inactive lanes must pass act=false (their result is unused).
__device__ __forceinline__ uint32_t peers_by_bits(uint32_t key, uint32_t nbits, bool act) {
    uint32_t peers = __ballot_sync(FULLMASK, act);
    for (uint32_t b = 0; b < nbits; ++b) {
        const bool bit = (key >> b) & 1u;
        const uint32_t m = __ballot_sync(FULLMASK, bit);
        peers &= bit ? m : ~m;
    }
    return peers;
}

// bit i of the result: slices i .. i+size-1 of `free16` are all free (log-step AND of shifted copies)
__device__ __forceinline__ uint32_t fit_map(uint32_t free16, uint32_t size) {
    uint32_t t = free16, r = size - 1u, s = 1u;
    while (r) { uint32_t m = s < r ? s : r; t &= t >> m; r -= m; s <<= 1; }
    return t;
}

__device__ __forceinline__ uint32_t meta(uint32_t start, uint32_t size, uint32_t prof, uint32_t st) {
    return start | (size << 8) | (prof << 16) | (st << 24);
}

// ---- one lane = one GPU of the node ---------------------------------------------------------------
struct Lane {
    uint32_t busy, flags, model, mem, share;
    bool valid;
    __device__ __forceinline__ void load(uint4 r, bool v) {
        valid = v;
        busy = v ? (r.x & 0xFFFFu) : 0xFFFFu;
        flags = v ? ((r.x >> 16) & 0xFFu) : DRA_GPU_UNAVAILABLE;
        model = v ? ((r.x >> 24) & 0xFu) : 0u;
        mem = v ? r.y : 0u;
        share = v ? (r.w & 0xFFFFu) : 0u;
    }
    __device__ __forceinline__ uint4 store(uint4 r) const {
        r.x = (r.x & 0xFF000000u) | (flags << 16) | busy;
        r.y = mem;
        r.w = (r.w & 0xFFFF0000u) | share;
        return r;
    }
};

// Per-warp monotone failure memo (spec §2: a batch only ever takes capacity, so a request shape that
// failed once on this node fails for the rest of the batch).  Lets failing claims skip the ballot.
struct Dead {
    uint32_t nocap = 0, bad = 0;     // per MIG profile
    uint32_t gpu_min = 0xFFFFu;      // smallest GPU count that failed
    uint64_t sh_min = 1ull << 32;    // smallest SHARED limit that failed
};

// Sink for Allocate: writes OutRecs.
struct OutSink {
    uint2* out; uint32_t n_out; Err err; uint32_t lane;
    // multi-GPU: every record is also appended to a queue in shared memory ({gpu, meta, slot, tag}, 16 B) from which the
    // CTA's idle warps send it to the peers WHILE the packing warp goes on (k_fused; 0 = no queue)
    uint32_t q_addr = 0, q_cap = 0, q_cnt = 0, q_tag = 0;
    __device__ __forceinline__ bool range(uint32_t dst, uint32_t slots) const {
        if (dst > n_out || slots > n_out - dst) { if (lane == 0) err.set(ERR_OUT_RANGE); return false; }
        return true;
    }
    __device__ __forceinline__ void put(uint32_t idx, uint32_t gpu, uint32_t m) const {
        out[idx] = make_uint2(gpu, m);
        if (q_addr) {                                       // one shared-memory atomic per group of converged lanes
            const uint32_t act = __activemask(), ldr = (uint32_t)__ffs(act) - 1u;
            uint32_t base = 0;
            if (lane == ldr) asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(base) : "r"(q_cnt), "r"((uint32_t)__popc(act)) : "memory");
            base = __shfl_sync(act, base, ldr);
            uint32_t ltm; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(ltm));
            const uint32_t pos = base + (uint32_t)__popc(act & ltm);
            if (pos < q_cap)
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(q_addr + (pos << 4)), "r"(gpu), "r"(m), "r"(idx), "r"(q_tag) : "memory");
        }
    }
    __device__ __forceinline__ bool in_range(uint32_t idx) const { return idx < n_out; }
    __device__ __forceinline__ void fail(uint32_t dst, uint32_t slots, uint32_t prof, uint32_t st) {
        if (lane < slots) put(dst + lane, DRA_GPU_NONE, meta(0, 0, prof, st));
    }
    __device__ __forceinline__ void mark_failed() {}
    __device__ __forceinline__ bool stop() const { return false; }
};

// Sink for UnsuitableNodes: only remembers whether anything failed.
struct FlagSink {
    bool failed = false;
    __device__ __forceinline__ bool range(uint32_t, uint32_t) const { return true; }
    __device__ __forceinline__ void put(uint32_t, uint32_t, uint32_t) const {}
    __device__ __forceinline__ bool in_range(uint32_t) const { return true; }
    __device__ __forceinline__ void fail(uint32_t, uint32_t, uint32_t, uint32_t) { failed = true; }
    __device__ __forceinline__ void mark_failed() { failed = true; }
    __device__ __forceinline__ bool stop() const { return failed; }
};

// ---- selectors (spec §10) ----------------------------------------------------------------------------
// GpuAttr as uint4: x memTotalMiB, y cc, z index, w product | driverMajor<<16.  Selector = 4 x uint4 (8 SelIns).
struct SelCtx { const uint4* attrs; const uint4* sels; uint32_t n_sel; };

__device__ __forceinline__ uint32_t claim_sel(uint32_t kind, uint32_t mem, uint32_t group) {
    return (kind == DRA_KIND_GPU || kind == DRA_KIND_MIG) ? mem : (kind == DRA_KIND_SHARED ? group : 0u);
}

// does GPU `gidx` pass selector `id`?  Postfix program over a boolean stack kept in a bit register.
__device__ __noinline__ bool sel_pass(const SelCtx sc, uint32_t id, uint32_t gidx, bool valid) {
    if (id == 0) return true;
    if (id > sc.n_sel || !valid) return false;
    uint4 a = make_uint4(0, 0, 0, 0);
    if (sc.attrs) a = __ldg(&sc.attrs[gidx]);
    uint32_t stack = 0, sp = 0; bool any = false, bad = false;
    #pragma unroll 1
    for (uint32_t q = 0; q < 4 && !bad; ++q) {
        const uint4 w = __ldg(&sc.sels[(size_t)(id - 1) * 4 + q]);
        const uint32_t hdr[2] = {w.x, w.z}, val[2] = {w.y, w.w};
        #pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t op = hdr[h] & 0xFFu, attr = (hdr[h] >> 8) & 0xFFu, cmp = (hdr[h] >> 16) & 0xFFu, v2 = val[h];
            if (op == DRA_SEL_END) { q = 4; break; }
            any = true;
            if (op == DRA_SEL_CMP) {
                uint32_t v = 0;
                if (attr == DRA_ATTR_MEMORY_MIB) v = a.x; else if (attr == DRA_ATTR_CC) v = a.y;
                else if (attr == DRA_ATTR_INDEX) v = a.z; else if (attr == DRA_ATTR_PRODUCT) v = a.w & 0xFFFFu;
                else if (attr == DRA_ATTR_DRIVER_MAJOR) v = a.w >> 16; else { bad = true; break; }
                bool r = false;
                if (cmp == DRA_CMP_EQ) r = v == v2; else if (cmp == DRA_CMP_NE) r = v != v2;
                else if (cmp == DRA_CMP_LT) r = v < v2; else if (cmp == DRA_CMP_LE) r = v <= v2;
                else if (cmp == DRA_CMP_GT) r = v > v2; else if (cmp == DRA_CMP_GE) r = v >= v2;
                else if (cmp == DRA_CMP_IN_MASK) r = v < 32u && ((v2 >> v) & 1u); else { bad = true; break; }
                stack |= (r ? 1u : 0u) << sp; ++sp;
            } else if (op == DRA_SEL_AND || op == DRA_SEL_OR) {
                if (sp < 2) { bad = true; break; }
                const uint32_t b_ = (stack >> (sp - 1)) & 1u, a_ = (stack >> (sp - 2)) & 1u;
                sp -= 2; stack &= (1u << sp) - 1u;
                stack |= (op == DRA_SEL_AND ? (a_ & b_) : (a_ | b_)) << sp; ++sp;
            } else if (op == DRA_SEL_NOT) {
                if (sp < 1) { bad = true; break; }
                stack ^= 1u << (sp - 1);
            } else { bad = true; break; }
        }
    }
    if (bad) return false;
    if (!any) return true;
    return sp >= 1 && ((stack >> (sp - 1)) & 1u);
}

__device__ __forceinline__ bool claim_invalid(uint32_t kind, uint32_t prof, uint32_t count, bool have_off) {
    if (kind > DRA_KIND_SHARED) return true;
    if (kind == DRA_KIND_GPU) return count == 0 || count > DRA_MAX_COUNT || (!have_off && count != 1);
    if (kind == DRA_KIND_MIG) return prof >= DRA_MAX_PROFILES;
    return false;
}

// One claim (or one co-location run starting at k) on the node held by this warp.  Returns the number of
// claims consumed.  `get(m)` returns claim m of the node's span (uniform address, all lanes).
template <class Get, class Sink>
__device__ __forceinline__ uint32_t node_step(Lane& L, Dead& D, uint32_t lane, uint32_t g0,
                                              const uint32_t* __restrict__ tbl_s, Get get, uint32_t k,
                                              uint32_t cnt, Sink& sink, bool have_off, const SelCtx sc,
                                              const uint32_t gmask = FULLMASK, const uint32_t gbase = 0) {
    // `lane` is the absolute lane; the node's GPUs sit on lanes gbase .. of the sub-warp group `gmask`
    // (the whole warp for the pack kernels; 8/16-lane groups in k_unsuitable).  Ballots are restricted to
    // the group, so __ffs(b)-1 is still the absolute lane of the lowest GPU.
    const uint4 c = get(k);
    const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
    const uint32_t dst = c.y, group = c.w;
    constexpr uint32_t BLOCKED = DRA_GPU_MIG_ENABLED | DRA_GPU_FULL_ALLOCATED | DRA_GPU_UNAVAILABLE;
    const uint32_t sel = claim_sel(kind, c.z, c.w);
    const uint32_t mem = kind == DRA_KIND_SHARED ? c.z : 0u;
    // a claim with a selector sees its own subset of GPUs: the node-wide failure memo does not apply to it
    const bool memo = sel == 0;
    const bool selok = sel == 0 ? true : sel_pass(sc, sel, g0 + lane - gbase, L.valid);

    if (claim_invalid(kind, prof, count, have_off) || sel > sc.n_sel) {   // spec §3, §10
        const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU
                          : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : prof;
        const uint32_t sl = (kind == DRA_KIND_GPU && !claim_invalid(kind, prof, count, have_off)) ? count : 1u;
        if (sink.range(dst, sl)) sink.fail(dst, sl, op, DRA_ST_INVALID);
        return 1;
    }

    if (kind == DRA_KIND_MIG && group == 0) {                       // spec §5
        if (!sink.range(dst, 1)) return 1;
        const uint32_t pbit = 1u << prof;
        if (memo && ((D.bad | D.nocap) & pbit)) {
            sink.fail(dst, 1, prof, (D.bad & pbit) ? DRA_ST_BAD_PROFILE : DRA_ST_NO_CAPACITY);
            return 1;
        }
        const uint32_t e = tbl_s[L.model * DRA_MAX_PROFILES + prof];
        const uint32_t smask = e >> 16, size = e & 0xFFu;
        const bool offers = L.valid && (L.flags & (DRA_GPU_MIG_ENABLED | DRA_GPU_UNAVAILABLE)) == DRA_GPU_MIG_ENABLED
                            && smask != 0 && selok;
        const bool elig = offers && !(L.flags & DRA_GPU_FULL_ALLOCATED);
        const uint32_t cand = elig ? (fit_map(~L.busy & 0xFFFFu, size) & smask) : 0u;
        const uint32_t b = (__ballot_sync(gmask, cand != 0) & gmask);
        if (b) {
            if (lane == (uint32_t)__ffs(b) - 1u) {                  // lowest GPU
                const uint32_t st = (uint32_t)__ffs(cand) - 1u;     // lowest start
                L.busy |= ((1u << size) - 1u) << st;
                sink.put(dst, g0 + lane - gbase, meta(st, size, prof, DRA_ST_OK));
            }
        } else {
            const bool any = (__ballot_sync(gmask, offers) & gmask) != 0;
            if (memo) { if (any) D.nocap |= pbit; else D.bad |= pbit; }
            sink.fail(dst, 1, prof, any ? DRA_ST_NO_CAPACITY : DRA_ST_BAD_PROFILE);
        }
        return 1;
    }

    if (kind == DRA_KIND_MIG) {                                     // spec §6: co-location run
        uint32_t e_ = k + 1;
        const uint32_t lim = (cnt - k) < DRA_MAX_GROUP ? cnt : k + DRA_MAX_GROUP;
        while (e_ < lim) {
            const uint4 cm = get(e_);
            const uint32_t km = cm.x & 0xFFu, pm = (cm.x >> 8) & 0xFFu;
            if (km != DRA_KIND_MIG || cm.w != group || pm >= DRA_MAX_PROFILES || cm.z > sc.n_sel) break;
            ++e_;
        }
        // every lane tries the whole run on a private copy of its own GPU
        uint32_t tb = L.busy;
        bool ok = L.valid && (L.flags & BLOCKED) == DRA_GPU_MIG_ENABLED && selok;     // the first member's selector
        for (uint32_t m = k; m < e_; ++m) {
            const uint32_t pm = (get(m).x >> 8) & 0xFFu;
            const uint32_t en = tbl_s[L.model * DRA_MAX_PROFILES + pm];
            const uint32_t sm = en >> 16, sz = en & 0xFFu;
            const uint32_t cd = sm ? (fit_map(~tb & 0xFFFFu, sz) & sm) : 0u;
            ok = ok && cd != 0;
            if (cd) tb |= ((1u << sz) - 1u) << ((uint32_t)__ffs(cd) - 1u);
        }
        const uint32_t b = (__ballot_sync(gmask, ok) & gmask);
        if (b) {
            if (lane == (uint32_t)__ffs(b) - 1u) {                  // winner replays and emits
                uint32_t nb = L.busy;
                for (uint32_t m = k; m < e_; ++m) {
                    const uint4 cm = get(m);
                    const uint32_t pm = (cm.x >> 8) & 0xFFu;
                    const uint32_t en = tbl_s[L.model * DRA_MAX_PROFILES + pm];
                    const uint32_t sm = en >> 16, sz = en & 0xFFu;
                    const uint32_t st = (uint32_t)__ffs(fit_map(~nb & 0xFFFFu, sz) & sm) - 1u;
                    nb |= ((1u << sz) - 1u) << st;
                    if (sink.in_range(cm.y)) sink.put(cm.y, g0 + lane - gbase, meta(st, sz, pm, DRA_ST_OK));
                }
                L.busy = nb;
            }
        } else {
            if (lane < e_ - k) {
                const uint4 cm = get(k + lane);
                if (sink.in_range(cm.y))
                    sink.put(cm.y, DRA_GPU_NONE, meta(0, 0, (cm.x >> 8) & 0xFFu, DRA_ST_GROUP));
            }
            sink.mark_failed();
        }
        // members whose slot is out of range
        for (uint32_t m = k; m < e_; ++m) (void)sink.range(get(m).y, 1);
        return e_ - k;
    }

    if (kind == DRA_KIND_GPU) {                                     // spec §4
        if (!sink.range(dst, count)) return 1;
        if (memo && count >= D.gpu_min) { sink.fail(dst, count, DRA_PROFILE_GPU, DRA_ST_NO_CAPACITY); return 1; }
        const bool elig = L.valid && !(L.flags & BLOCKED) && L.share == 0 && selok;
        const uint32_t b = (__ballot_sync(gmask, elig) & gmask);
        if ((uint32_t)__popc(b) >= count) {
            const uint32_t r = (uint32_t)__popc(b & lanemask_lt());
            if (elig && r < count) {
                L.flags |= DRA_GPU_FULL_ALLOCATED;
                sink.put(dst + r, g0 + lane - gbase, meta(0, 0, DRA_PROFILE_GPU, DRA_ST_OK));
            }
        } else {
            if (memo) D.gpu_min = count;
            sink.fail(dst, count, DRA_PROFILE_GPU, DRA_ST_NO_CAPACITY);
        }
        return 1;
    }

    // SHARED, spec §7
    if (!sink.range(dst, 1)) return 1;
    if (memo && (uint64_t)mem >= D.sh_min) { sink.fail(dst, 1, DRA_PROFILE_SHARED, DRA_ST_MEM_LIMIT); return 1; }
    {
        const bool elig = L.valid && !(L.flags & BLOCKED) && L.share < 0xFFFFu && L.mem >= mem && selok;
        const uint32_t b = (__ballot_sync(gmask, elig) & gmask);
        if (b) {
            if (lane == (uint32_t)__ffs(b) - 1u) {
                L.mem -= mem; L.share += 1;
                sink.put(dst, g0 + lane - gbase, meta(0, 0, DRA_PROFILE_SHARED, DRA_ST_OK));
            }
        } else {
            if (memo) D.sh_min = mem;
            sink.fail(dst, 1, DRA_PROFILE_SHARED, DRA_ST_MEM_LIMIT);
        }
    }
    return 1;
}

// Out-of-line copy for the pack kernels: co-location runs are rare there, and keeping ~900 instructions out
// of the hot loop's instruction-cache footprint matters more than the call (the kernel runs once per SM).
template <class Get, class Sink>
__device__ __noinline__ uint32_t node_step_cold(Lane& L, Dead& D, uint32_t lane, uint32_t g0,
                                                const uint32_t* __restrict__ tbl_s, Get get, uint32_t k,
                                                uint32_t cnt, Sink& sink, bool have_off, const SelCtx sc) {
    return node_step(L, D, lane, g0, tbl_s, get, k, cnt, sink, have_off, sc);
}

// ====================================================================================================
// bucketing: stable counting sort of claims by node
// ====================================================================================================

// grid = n_tiles, block = 32.  Tile t owns claims [t*T, (t+1)*T).  Dynamic smem: (n_node+1) u16 counters.
// hist[t][n] = number of tile-t claims on node n (bucket n_node = claims naming no node);
// rank[i]    = number of earlier claims of the same tile with the same node (stable rank).
__global__ void __launch_bounds__(32)
k_bucket_hist(const uint4* __restrict__ claims, uint32_t n_claim, uint32_t n_node, uint32_t T,
              uint32_t* __restrict__ hist, uint16_t* __restrict__ rank) {
    extern __shared__ uint16_t cnt[];
    pdl_trigger();
    const uint32_t lane = threadIdx.x, nb = n_node + 1;
    const uint32_t nbits = 32u - (uint32_t)__clz(n_node);          // keys are 0..n_node
    for (uint32_t n = lane; n < nb; n += 32) cnt[n] = 0;
    __syncwarp();
    const uint32_t base = blockIdx.x * T;
    const uint32_t end = min(n_claim, base + T);
    for (uint32_t i0 = base; i0 < end; i0 += 32) {
        const uint32_t i = i0 + lane;
        const bool act = i < end;
        uint32_t key = 0xFFFFFFFFu;
        if (act) { key = __ldg(&claims[i]).y; key = key < n_node ? key : n_node; }
        const uint32_t m = peers_by_bits(key, nbits, act);
        const uint32_t r = (uint32_t)__popc(m & lanemask_lt());
        uint32_t old = 0;
        if (act) { old = cnt[key]; rank[i] = (uint16_t)(old + r); }
        __syncwarp();
        if (act && r == 0) cnt[key] = (uint16_t)(old + (uint32_t)__popc(m));
        __syncwarp();
    }
    uint32_t* h = hist + (size_t)blockIdx.x * nb;
    for (uint32_t n = lane; n < nb; n += 32) h[n] = cnt[n];
}

// one CTA of 1024 threads.  In place: hist[t][n] <- sum_{t' < t} hist[t'][n];
// claim_off[n] <- sum_{n' < n} total[n'] for n in [0, n_node+1]  (claim_off[n_node+1] = n_claim).
__global__ void __launch_bounds__(1024)
k_bucket_scan(uint32_t* __restrict__ hist, uint32_t n_tiles, uint32_t n_node,
              uint32_t* __restrict__ claim_off) {
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry_s, total_s;
    const uint32_t nb = n_node + 1, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    pdl_trigger(); pdl_wait();
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (uint32_t n0 = 0; n0 < nb; n0 += 1024) {
        const uint32_t n = n0 + tid;
        uint32_t run = 0;
        if (n < nb) {
            uint32_t t = 0;
            for (; t + 4 <= n_tiles; t += 4) {
                uint32_t* p = hist + (size_t)t * nb + n;
                const uint32_t v0 = p[0], v1 = p[nb], v2 = p[2 * (size_t)nb], v3 = p[3 * (size_t)nb];
                p[0] = run; run += v0; p[nb] = run; run += v1;
                p[2 * (size_t)nb] = run; run += v2; p[3 * (size_t)nb] = run; run += v3;
            }
            for (; t < n_tiles; ++t) { uint32_t* p = hist + (size_t)t * nb + n; const uint32_t v = *p; *p = run; run += v; }
        }
        // block-wide exclusive scan of `run`
        uint32_t x = run;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) wsum[wid] = x;
        __syncthreads();
        if (wid == 0) {
            const uint32_t w = wsum[lane];
            uint32_t ws = w;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, ws, d); if (lane >= (uint32_t)d) ws += y; }
            wsum[lane] = ws - w;                       // exclusive warp offsets
            if (lane == 31) total_s = ws;
        }
        __syncthreads();
        const uint32_t excl = carry_s + wsum[wid] + (x - run);
        if (n < nb) claim_off[n] = excl;
        __syncthreads();
        if (tid == 0) carry_s += total_s;
        __syncthreads();
    }
    if (tid == 0) claim_off[nb] = carry_s;
}

// ---- CTA-wide tiles (used whenever 8*(n_node+1) u16 counters fit in shared memory) ----------------------------
// k_bucket_hist8: grid = n_tiles, 256 threads; tile = 2048 claims, warp w owns rows w*8 .. w*8+7 of it.
// Per-warp counters keep the pass stable (as k_bucket_small); all 8 keys of a lane are loaded before the first
// is used.  hist[t][n] = claims of tile t on node n; rank[i] = stable rank of claim i inside its tile.
constexpr uint32_t H8_TILE = 2048;
template <bool MULTI>
__global__ void __launch_bounds__(256)
k_bucket_hist8(const uint4* __restrict__ claims, uint32_t n_claim, uint32_t n_node,
               uint32_t* __restrict__ hist, uint16_t* __restrict__ rank, const uint32_t* __restrict__ n_dev, const uint32_t T) {
    extern __shared__ uint16_t cnt8[];                              // [8][nbp]
    pdl_trigger();
    if (n_dev) n_claim = min(n_claim, __ldcg(n_dev));               // sharded call: compacted on the device
    const uint32_t nb = n_node + 1, nbp = (nb + 1) & ~1u;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t nbits = 32u - (uint32_t)__clz(n_node);
    if (MULTI) {
        // Large batches (T = m x 2048, chosen so that the tiles fill the SMs once): the per-tile work that is
        // proportional to the number of NODES (clearing 8 counter rows, combining them, one hist row out — and a
        // column of the matrix for the scan and the scatter to walk) is paid once per T claims instead of once per
        // 2048.  A warp owns T/8 consecutive claims and walks them 8 rows at a time; the ranks inside the warp's part
        // go out as they are found, the warp's base inside the tile is added in a second sweep (keys re-read: L2 hits).
        const uint32_t per_warp = T >> 3, w0 = blockIdx.x * T + wid * per_warp;
        for (uint32_t i = tid; i < 4 * nbp; i += 256) reinterpret_cast<uint32_t*>(cnt8)[i] = 0;
        __syncthreads();
        uint16_t* mycnt = cnt8 + wid * nbp;
        uint32_t* row32 = reinterpret_cast<uint32_t*>(mycnt);             // (nbp is even: every warp's row starts on a word)
        for (uint32_t c0 = 0; c0 < per_warp; c0 += 256) {
            uint32_t keys[8];
            #pragma unroll
            for (int r = 0; r < 8; ++r) { const uint32_t i = w0 + c0 + r * 32 + lane; keys[r] = i < n_claim ? __ldg(&claims[i]).y : 0xFFFFFFFFu; }
            #pragma unroll
            for (int r = 0; r < 8; ++r) {
                const uint32_t i = w0 + c0 + r * 32 + lane;
                const bool act = i < n_claim;
                const uint32_t key = act ? (keys[r] < n_node ? keys[r] : n_node) : 0u;
                // the row's 32 keys are almost always distinct (32 of thousands of nodes): a shared-memory atomic on the
                // u16 counter (the half of a 32-bit word) hands every lane its rank in one instruction; only if two lanes
                // of the row share a key — the count grew by more than one — does the hardware's order among them have
                // to be replaced by lane order, with the votes that otherwise cost ~70 instructions per row
                const uint32_t sh = (key & 1u) << 4;
                uint32_t old = 0;
                if (act) old = (atomicAdd(&row32[key >> 1], 1u << sh) >> sh) & 0xFFFFu;
                __syncwarp();
                const uint32_t now = act ? (row32[key >> 1] >> sh) & 0xFFFFu : 0u;
                if (__any_sync(FULLMASK, act && now != old + 1u)) {
                    const uint32_t m = peers_by_bits(key, nbits, act);
                    old = now - (uint32_t)__popc(m) + (uint32_t)__popc(m & lanemask_lt());
                }
                if (act) rank[i] = (uint16_t)old;
                __syncwarp();
            }
        }
        __syncthreads();
        uint32_t* h = hist + (size_t)blockIdx.x * nb;
        for (uint32_t n = tid; n < nb; n += 256) {
            uint32_t run = 0;
            #pragma unroll
            for (uint32_t w = 0; w < 8; ++w) { const uint32_t v = cnt8[w * nbp + n]; cnt8[w * nbp + n] = (uint16_t)run; run += v; }
            h[n] = run;
        }
        __syncthreads();
        if (wid != 0)                                               // (warp 0's base is zero everywhere)
            for (uint32_t c0 = 0; c0 < per_warp; c0 += 256) {
                uint32_t keys[8];
                #pragma unroll
                for (int r = 0; r < 8; ++r) { const uint32_t i = w0 + c0 + r * 32 + lane; keys[r] = i < n_claim ? __ldg(&claims[i]).y : 0xFFFFFFFFu; }
                #pragma unroll
                for (int r = 0; r < 8; ++r) {
                    const uint32_t i = w0 + c0 + r * 32 + lane;
                    if (i < n_claim) rank[i] = (uint16_t)(rank[i] + mycnt[keys[r] < n_node ? keys[r] : n_node]);
                }
            }
        return;
    }
    const uint32_t w0 = blockIdx.x * H8_TILE + wid * 256;
    uint32_t keys[8];
    #pragma unroll
    for (int r = 0; r < 8; ++r) { const uint32_t i = w0 + r * 32 + lane; keys[r] = i < n_claim ? __ldg(&claims[i]).y : 0xFFFFFFFFu; }
    for (uint32_t i = tid; i < 4 * nbp; i += 256) reinterpret_cast<uint32_t*>(cnt8)[i] = 0;
    __syncthreads();
    uint16_t* mycnt = cnt8 + wid * nbp;
    uint32_t* row32 = reinterpret_cast<uint32_t*>(mycnt);
    uint32_t local[8];
    #pragma unroll
    for (int r = 0; r < 8; ++r) {
        const uint32_t i = w0 + r * 32 + lane;
        const bool act = i < n_claim;
        const uint32_t key = act ? (keys[r] < n_node ? keys[r] : n_node) : 0u;
        keys[r] = key;
        // (as above: an atomic on the u16 half-word gives the rank; votes only for a row in which two lanes share a node)
        const uint32_t sh = (key & 1u) << 4;
        uint32_t old = 0;
        if (act) old = (atomicAdd(&row32[key >> 1], 1u << sh) >> sh) & 0xFFFFu;
        __syncwarp();
        const uint32_t now = act ? (row32[key >> 1] >> sh) & 0xFFFFu : 0u;
        if (__any_sync(FULLMASK, act && now != old + 1u)) {
            const uint32_t m = peers_by_bits(key, nbits, act);
            old = now - (uint32_t)__popc(m) + (uint32_t)__popc(m & lanemask_lt());
        }
        local[r] = old;
        __syncwarp();
    }
    __syncthreads();
    uint32_t* h = hist + (size_t)blockIdx.x * nb;
    for (uint32_t n = tid; n < nb; n += 256) {
        uint32_t run = 0;
        #pragma unroll
        for (uint32_t w = 0; w < 8; ++w) { const uint32_t v = cnt8[w * nbp + n]; cnt8[w * nbp + n] = (uint16_t)run; run += v; }
        h[n] = run;
    }
    __syncthreads();
    #pragma unroll
    for (int r = 0; r < 8; ++r) {
        const uint32_t i = w0 + r * 32 + lane;
        if (i < n_claim) rank[i] = (uint16_t)(mycnt[keys[r]] + local[r]);
    }
}

// The last CTA of a scan kernel (256 threads): node totals in claim_off[0..nb) -> exclusive offsets, claim_off[nb] = sum.
// Thread t owns a contiguous run of ceil(nb/256) nodes: one sweep to sum them (8 loads in flight), ONE block-wide scan of
// the 256 sums, one sweep to write — the number of dependent round trips does not grow with the number of nodes (a
// round per 256 nodes would).
__device__ __forceinline__ void totals_to_offsets(uint32_t* __restrict__ claim_off, const uint32_t nb, uint32_t* wsum /* [9] shared */) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t per = (nb + 255) / 256, lo = min(nb, tid * per), hi = min(nb, lo + per);
    uint32_t sum = 0, m = lo;
    for (; m + 8 <= hi; m += 8) {
        uint32_t v[8];
        #pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = __ldcg(&claim_off[m + q]);
        #pragma unroll
        for (int q = 0; q < 8; ++q) sum += v[q];
    }
    for (; m < hi; ++m) sum += __ldcg(&claim_off[m]);
    uint32_t x = sum;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, x, d); if (lane >= (uint32_t)d) x += y; }
    __syncthreads();                                   // (wsum may still be read by a previous use)
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        const uint32_t w = lane < 8 ? wsum[lane] : 0u;
        uint32_t ws = w;
        #pragma unroll
        for (int d = 1; d < 8; d <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, ws, d); if (lane >= (uint32_t)d) ws += y; }
        __syncwarp();
        if (lane < 8) wsum[lane] = ws - w;
        if (lane == 7) wsum[8] = ws;
    }
    __syncthreads();
    uint32_t run = wsum[wid] + (x - sum);
    m = lo;
    for (; m + 8 <= hi; m += 8) {
        uint32_t v[8];
        #pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = __ldcg(&claim_off[m + q]);
        #pragma unroll
        for (int q = 0; q < 8; ++q) { claim_off[m + q] = run; run += v[q]; }
    }
    for (; m < hi; ++m) { const uint32_t v = __ldcg(&claim_off[m]); claim_off[m] = run; run += v; }
    if (tid == 0) claim_off[nb] = wsum[8];
}

// k_bucket_scan8: grid = ceil((n_node+1)/8) CTAs of 8 warps, WARP per node, lanes over the tiles: every load of a
// node's column is in flight at once (the thread-per-node form walked the tiles in 7 dependent L2 round trips on 4
// SMs), the prefix over the tiles is a warp scan by shuffles.  In place: hist[t][n] <- sum_{t'<t}; node totals go to
// claim_off[n]; the LAST CTA to finish (ticket) turns the totals into the exclusive offsets.
__global__ void __launch_bounds__(256)
k_bucket_scan8(uint32_t* __restrict__ hist, uint32_t n_tiles, uint32_t n_node, uint32_t* __restrict__ claim_off,
               uint32_t* __restrict__ ticket) {
    const uint32_t nb = n_node + 1, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    pdl_trigger(); pdl_wait();
    const uint32_t n = blockIdx.x * 8 + wid;
    if (n < nb) {
        uint32_t run = 0;
        for (uint32_t t0 = 0; t0 < n_tiles; t0 += 128) {                   // 4 tiles per lane and round
            uint32_t v[4], x[4];
            #pragma unroll
            for (int q = 0; q < 4; ++q) { const uint32_t t = t0 + q * 32 + lane; v[q] = t < n_tiles ? __ldcg(&hist[(size_t)t * nb + n]) : 0u; }
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                x[q] = v[q];
                #pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULLMASK, x[q], d); if (lane >= (uint32_t)d) x[q] += y; }
            }
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint32_t t = t0 + q * 32 + lane;
                if (t < n_tiles) hist[(size_t)t * nb + n] = run + x[q] - v[q];
                run += __shfl_sync(FULLMASK, x[q], 31);
            }
        }
        if (lane == 0) claim_off[n] = run;
    }
    __threadfence();
    __shared__ uint32_t last_s, wsum[9];
    __syncthreads();
    if (tid == 0) last_s = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (!last_s) return;
    if (tid == 0) *ticket = 0;
    __threadfence();
    totals_to_offsets(claim_off, nb, wsum);
}

// k_bucket_scan_rows: the same scan for BIG matrices (n_tiles x nb beyond ~0.5M counters), where the warp-per-node form
// above drags a 32-byte sector through L2 for every 4-byte counter, twice (at 1M claims on 10k nodes, most of the
// batch).  Here a CTA owns 32 consecutive nodes, lane = node, and every access is a coalesced 128-byte row piece:
// warp w sums its share of the tiles (8 loads in flight), the warps' sums are combined in shared memory, and a second
// sweep (L2 hits) writes the exclusive prefixes.  Node totals -> claim_off; the last CTA (ticket) makes them offsets.
__global__ void __launch_bounds__(256)
k_bucket_scan_rows(uint32_t* __restrict__ hist, uint32_t n_tiles, uint32_t n_node, uint32_t* __restrict__ claim_off,
                   uint32_t* __restrict__ ticket, unsigned long long* __restrict__ status, Err err) {
    const uint32_t nb = n_node + 1, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    __shared__ uint32_t part[8][32];
    pdl_trigger(); pdl_wait();
    // this launch's epoch: a device word that the LAST CTA to finish advances (so a replayed CUDA graph gets a new one too);
    // nobody can have advanced it before every CTA has read it, because the last ticket is taken after all of them started
    const uint32_t epoch = __ldcg(ticket + 1) + 1u;
    const uint32_t n = blockIdx.x * 32 + lane;
    const uint32_t K = (n_tiles + 7) / 8, t_lo = min(n_tiles, wid * K), t_hi = min(n_tiles, t_lo + K);
    uint32_t sum = 0;
    if (n < nb) {
        uint32_t t = t_lo;
        for (; t + 8 <= t_hi; t += 8) {
            uint32_t v[8];
            #pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = __ldcg(&hist[(size_t)(t + q) * nb + n]);
            #pragma unroll
            for (int q = 0; q < 8; ++q) sum += v[q];
        }
        for (; t < t_hi; ++t) sum += __ldcg(&hist[(size_t)t * nb + n]);
    }
    part[wid][lane] = sum;
    __syncthreads();
    uint32_t run = 0, total = 0;
    #pragma unroll
    for (uint32_t w = 0; w < 8; ++w) { const uint32_t v = part[w][lane]; run += w < wid ? v : 0u; total += v; }
    if (wid == 0) {
        // node totals -> claim offsets without a serial tail: this CTA publishes the sum of its 32 nodes and adds up the
        // sums of ALL its predecessors (every load in flight at once, spinning only until the last of them is there)
        uint32_t x = total;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULLMASK, x, d); if (lane >= (uint32_t)d) x += y; }
        const uint32_t agg = __shfl_sync(FULLMASK, x, 31);
        if (lane == 0) atomicExch(&status[blockIdx.x], ((unsigned long long)epoch << 32) | agg);
        uint32_t base = 0;
        const long long t0 = clock64();
        bool dead = false;
        for (uint32_t b0 = 0; b0 < blockIdx.x && !dead; b0 += 256) {
            unsigned long long v[8];
            bool ready;
            do {
                ready = true;
                #pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint32_t idx = b0 + k * 32 + lane;
                    v[k] = 0;
                    if (idx < blockIdx.x) asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v[k]) : "l"(status + idx) : "memory");
                }
                #pragma unroll
                for (int k = 0; k < 8; ++k) if (b0 + k * 32 + lane < blockIdx.x && (uint32_t)(v[k] >> 32) != epoch) ready = false;
                if (clock64() - t0 > 2000000000ll) dead = true;
            } while (!__all_sync(FULLMASK, ready || dead));
            #pragma unroll
            for (int k = 0; k < 8; ++k) if (b0 + k * 32 + lane < blockIdx.x) base += (uint32_t)v[k];
        }
        base = __reduce_add_sync(FULLMASK, base);
        if (dead && lane == 0) err.set(ERR_DEVICE_WAIT);
        if (n < nb) claim_off[n] = base + x - total;
        if (blockIdx.x == gridDim.x - 1 && lane == 31) claim_off[nb] = base + agg;
    }
    if (n < nb) {
        uint32_t t = t_lo;
        for (; t + 8 <= t_hi; t += 8) {
            uint32_t v[8];
            #pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = __ldcg(&hist[(size_t)(t + q) * nb + n]);
            #pragma unroll
            for (int q = 0; q < 8; ++q) { hist[(size_t)(t + q) * nb + n] = run; run += v[q]; }
        }
        for (; t < t_hi; ++t) { const uint32_t v = __ldcg(&hist[(size_t)t * nb + n]); hist[(size_t)t * nb + n] = run; run += v; }
    }
    __syncthreads();
    if (tid == 0 && atomicAdd(ticket, 1u) == gridDim.x - 1) { *ticket = 0; __threadfence(); atomicAdd(ticket + 1, 1u); }
}

// thread per claim.  sorted[dest] = claim with .y replaced by its first OutRec slot.
// Claims that name no node (bucket n_node) get their INVALID record here and are not sorted in.
__global__ void __launch_bounds__(256)
k_bucket_scatter(const uint4* __restrict__ claims, uint32_t n_claim, uint32_t n_node, uint32_t T,
                 const uint32_t* __restrict__ hist, const uint16_t* __restrict__ rank,
                 const uint32_t* __restrict__ claim_off, const uint32_t* __restrict__ out_off,
                 uint4* __restrict__ sorted, uint2* __restrict__ out, uint32_t n_out, Err err, const uint32_t* __restrict__ n_dev) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (n_dev) n_claim = min(n_claim, __ldcg(n_dev));
    if (i >= n_claim) { pdl_trigger(); return; }
    uint4 c = __ldg(&claims[i]);
    const uint32_t dst = out_off ? __ldg(&out_off[i]) : i;
    pdl_trigger(); pdl_wait();                             // the inputs above do not come from the chain
    const uint32_t nb = n_node + 1;
    if (c.y >= n_node) {
        const uint32_t kind = c.x & 0xFFu;
        const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU
                          : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : ((c.x >> 8) & 0xFFu);
        if (!out) return;                                  // pod records (k_pod_records has reported them)
        if (dst < n_out) out[dst] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, DRA_ST_INVALID));
        else err.set(ERR_OUT_RANGE);
        return;
    }
    const uint32_t t = i / T;
    const uint32_t dest = __ldg(&claim_off[c.y]) + __ldg(&hist[(size_t)t * nb + c.y]) + rank[i];
    c.y = dst;
    sorted[dest] = c;
}

// What later kernels of the batch will read: pulled into L2 by the first kernel so that the pack kernel's
// dependent round trips are L2 hits, not DRAM misses (cp.async.bulk.prefetch.L2).
struct Prefetch { const void* p[3]; uint32_t bytes[3]; };

// Whole stable counting sort in ONE CTA of 1024 threads, for batches that fit (n_claim <= 32768 and
// 32*(n_node+1) u16 counters + n_claim u16 ranks in shared memory).  Replaces hist+scan+scatter by one launch:
//   warp w owns claims [w*R*32, (w+1)*R*32) (R rows of 32);  per-warp counters keep the pass stable.
// Loads are issued 16 rows at a time before any of them is used (cold-DRAM latency paid once per chunk).
// Dynamic smem layout: u32 off[nb] | u16 cnt[32][nb] | u16 rank[n_claim]
constexpr int BS_CHUNK = 16;
__global__ void __launch_bounds__(1024)
k_bucket_small(const uint4* __restrict__ claims, uint32_t n_claim, uint32_t n_node,
               const uint32_t* __restrict__ out_off, uint32_t* __restrict__ claim_off,
               uint4* __restrict__ sorted, uint2* __restrict__ out, uint32_t n_out, Err err, Prefetch pf,
               const uint32_t* __restrict__ n_dev) {
    extern __shared__ uint32_t sm_u32[];
    pdl_trigger();
    if (n_dev) n_claim = min(n_claim, __ldcg(n_dev));
    const uint32_t nb = n_node + 1, nbp = (nb + 1) & ~1u;
    uint32_t* off = sm_u32;                                        // [nbp]
    uint16_t* cnt = reinterpret_cast<uint16_t*>(off + nbp);        // [32][nbp]
    uint16_t* rnk = cnt + 32 * nbp;                                // [n_claim]
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry_s, total_s;
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

    if (tid == 0 && pf.bytes[0]) tma_prefetch_l2(pf.p[0], pf.bytes[0]);
    if (tid == 32 && pf.bytes[1]) tma_prefetch_l2(pf.p[1], pf.bytes[1]);
    if (tid == 64 && pf.bytes[2]) tma_prefetch_l2(pf.p[2], pf.bytes[2]);

    const uint32_t R = (n_claim + 1023) / 1024;                    // rows per warp
    const uint32_t w0 = wid * R * 32;
    uint16_t* mycnt = cnt + wid * nbp;
    const uint32_t nbits = 32u - (uint32_t)__clz(n_node);          // keys are 0..n_node

    // first chunk of keys in flight while the counters are cleared
    uint32_t keys[BS_CHUNK];
    #pragma unroll
    for (int q = 0; q < BS_CHUNK; ++q) {
        const uint32_t i = w0 + q * 32 + lane;
        keys[q] = ((uint32_t)q < R && i < n_claim) ? __ldg(&claims[i]).y : 0xFFFFFFFFu;
    }
    for (uint32_t i = tid; i < 16 * nbp; i += 1024) reinterpret_cast<uint32_t*>(cnt)[i] = 0;
    if (tid == 0) carry_s = 0;
    __syncthreads();

    for (uint32_t r0 = 0; r0 < R; r0 += BS_CHUNK) {
        if (r0) {
            #pragma unroll
            for (int q = 0; q < BS_CHUNK; ++q) {
                const uint32_t i = w0 + (r0 + q) * 32 + lane;
                keys[q] = (r0 + q < R && i < n_claim) ? __ldg(&claims[i]).y : 0xFFFFFFFFu;
            }
        }
        #pragma unroll
        for (int q = 0; q < BS_CHUNK; ++q) {
            if (r0 + q < R) {                                       // warp-uniform
                const uint32_t i = w0 + (r0 + q) * 32 + lane;
                const bool act = i < n_claim;
                const uint32_t key = act ? (keys[q] < n_node ? keys[q] : n_node) : 0xFFFFFFFFu;
                const uint32_t m = peers_by_bits(key, nbits, act);
                const uint32_t rk = (uint32_t)__popc(m & lanemask_lt());
                uint32_t old = 0;
                if (act) { old = mycnt[key]; rnk[i] = (uint16_t)(old + rk); }
                __syncwarp();
                if (act && rk == 0) mycnt[key] = (uint16_t)(old + (uint32_t)__popc(m));
                __syncwarp();
            }
        }
    }
    __syncthreads();

    // per node: exclusive scan over the 32 warps' counters, then block scan of node totals
    for (uint32_t n0 = 0; n0 < nb; n0 += 1024) {
        const uint32_t n = n0 + tid;
        uint32_t run = 0;
        if (n < nb) {
            #pragma unroll 8
            for (uint32_t w = 0; w < 32; ++w) { const uint32_t v = cnt[w * nbp + n]; cnt[w * nbp + n] = (uint16_t)run; run += v; }
        }
        uint32_t x = run;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) wsum[wid] = x;
        __syncthreads();
        if (wid == 0) {
            const uint32_t w = wsum[lane];
            uint32_t ws = w;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(FULLMASK, ws, d); if (lane >= (uint32_t)d) ws += y; }
            wsum[lane] = ws - w;
            if (lane == 31) total_s = ws;
        }
        __syncthreads();
        const uint32_t excl = carry_s + wsum[wid] + (x - run);
        if (n < nb) { off[n] = excl; claim_off[n] = excl; }
        __syncthreads();
        if (tid == 0) carry_s += total_s;
        __syncthreads();
    }
    if (tid == 0) claim_off[nb] = carry_s;

    // scatter: claims come back from L2 now; again all loads of a chunk before the first use
    for (uint32_t r0 = 0; r0 < R; r0 += BS_CHUNK / 2) {
        uint4 cc[BS_CHUNK / 2]; uint32_t dd[BS_CHUNK / 2];
        #pragma unroll
        for (int q = 0; q < BS_CHUNK / 2; ++q) {
            const uint32_t i = w0 + (r0 + q) * 32 + lane;
            const bool act = r0 + q < R && i < n_claim;
            cc[q] = act ? __ldg(&claims[i]) : make_uint4(0, 0, 0, 0);
            dd[q] = act ? (out_off ? __ldg(&out_off[i]) : i) : 0;
        }
        #pragma unroll
        for (int q = 0; q < BS_CHUNK / 2; ++q) {
            const uint32_t i = w0 + (r0 + q) * 32 + lane;
            if (r0 + q >= R || i >= n_claim) continue;
            uint4 c = cc[q];
            const uint32_t dst = dd[q];
            if (c.y >= n_node) {
                const uint32_t kind = c.x & 0xFFu;
                const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU
                                  : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : ((c.x >> 8) & 0xFFu);
                if (!out) continue;                        // pod records
                if (dst < n_out) out[dst] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, DRA_ST_INVALID));
                else err.set(ERR_OUT_RANGE);
                continue;
            }
            const uint32_t dest = off[c.y] + mycnt[c.y] + rnk[i];
            c.y = dst;
            sorted[dest] = c;
        }
    }
}

// DRA_F_NODE_SORTED input: verify order, build claim_off by boundary detection, copy with slot embedded.
__global__ void __launch_bounds__(256)
k_sorted_prep(const uint4* __restrict__ claims, uint32_t n_claim, uint32_t n_node,
              const uint32_t* __restrict__ out_off, uint32_t* __restrict__ claim_off,
              uint4* __restrict__ sorted, uint2* __restrict__ out, uint32_t n_out, Err err) {
    pdl_trigger();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && n_claim == 0) { for (uint32_t n = 0; n <= n_node + 1; ++n) claim_off[n] = 0; }
    if (i >= n_claim) return;
    uint4 c = __ldg(&claims[i]);
    const uint32_t key = c.y < n_node ? c.y : n_node;
    uint32_t prev = 0; bool first = i == 0;
    if (!first) { prev = __ldg(&claims[i - 1]).y; prev = prev < n_node ? prev : n_node; }
    if (!first && prev > key) err.set(ERR_NOT_SORTED);
    // claim_off[n] = i for every bucket n in (prev, key]  (first claim: [0, key])
    if (first) { for (uint32_t n = 0; n <= key; ++n) claim_off[n] = 0; }
    else if (prev < key) { for (uint32_t n = prev + 1; n <= key; ++n) claim_off[n] = i; }
    if (i == n_claim - 1) { for (uint32_t n = key + 1; n <= n_node + 1; ++n) claim_off[n] = n_claim; }
    const uint32_t dst = out_off ? __ldg(&out_off[i]) : i;
    if (key == n_node) {
        const uint32_t kind = c.x & 0xFFu;
        const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU
                          : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : ((c.x >> 8) & 0xFFu);
        if (dst < n_out) out[dst] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, DRA_ST_INVALID));
        else err.set(ERR_OUT_RANGE);
    }
    c.y = dst;
    sorted[i] = c;
}

// ====================================================================================================
// sharded global batch: every rank reads the WHOLE claim array and keeps the claims of its own node range
// ====================================================================================================
// (pool = node: vendor/k8s.io/dynamic-resource-allocation/kubeletplugin/draplugin.go:427-435 — nodes are sharded whole.)
// Stable compaction in one pass: tiles of 2048 claims, taken by ticket; a tile's prefix comes from a decoupled
// look-back over the earlier tiles' status words (state | epoch | claims | slots in ONE 64-bit word, so no fence).
// Kept claims are rewritten with the node index LOCAL to the shard; claims naming no node go to the rank with
// take_stray set (they come back INVALID, spec §3).  coff[j] = first GLOBAL OutRec slot of kept claim j.
__device__ __forceinline__ unsigned long long globaltimer_ns();
constexpr uint32_t SC_TILE = 2048;
constexpr int SC_IN_ROWS = 4;             // in-kernel form: tiles of 1024 claims, one per CTA of k_fused
struct ShardArgs {
    const uint4* claims; uint32_t n_claim; const uint32_t* out_off;
    uint32_t node_lo, node_hi, n_node_global, take_stray, have_off;
    uint4* cclaims; uint32_t* coff; uint32_t cap;
    unsigned long long* status; uint32_t* ticket; uint32_t n_tiles, epoch;
    uint32_t* counts;                 // [0] claims kept, [1] their OutRec slots
    volatile uint32_t* h_counts;      // the same, mapped host memory (plan hint for the next call)
    // every rank reads the WHOLE array, so it can count what each rank will answer: the gather then needs no header
    uint32_t world, stray_rank;       // world == 0: not counted
    uint32_t rank_hi[PEER_MAX];       // rank r serves nodes [rank_hi[r-1], rank_hi[r])
    uint32_t* rank_slots;             // [2][PEER_MAX] by epoch parity: OutRec slots per rank
    unsigned long long* timeline;     // instrumentation: [0] first CTA in, [1] last CTA out (globaltimer), or NULL
    Err err;
};
__device__ __forceinline__ unsigned long long sc_pack(uint32_t epoch, uint32_t state, uint32_t c, uint32_t s_) {
    return ((unsigned long long)state << 62) | ((unsigned long long)(epoch & 0x3FFu) << 52) | ((unsigned long long)(c & 0x3FFFFFFu) << 26) | (s_ & 0x3FFFFFFu);
}
__global__ void __launch_bounds__(256)
k_shard_compact(const ShardArgs a) {
    __shared__ uint32_t tile_s, rowc[64], rows[64], pre_c, pre_s, rs_s[PEER_MAX];
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, ltm = lanemask_lt();
    pdl_trigger();                                           // the allocation kernel's prologue may overlap this kernel
    if (a.timeline && tid == 0) atomicMin(a.timeline, globaltimer_ns());
    if (tid < PEER_MAX) rs_s[tid] = 0;
    if (tid == 0) {
        const uint32_t t = atomicAdd(a.ticket, 1u);
        if (t == a.n_tiles - 1) *a.ticket = 0;                    // the last ticket of this launch: ready for the next
        tile_s = t;
    }
    __syncthreads();
    const uint32_t tile = tile_s;
    const uint32_t w0 = tile * SC_TILE + wid * 256;
    uint4 c[8]; uint32_t keepm = 0, rk[8];
    uint32_t own_sl[8];                                      // owner rank << 16 | slots, of every claim of the tile (world > 0)
    #pragma unroll
    for (int r = 0; r < 8; ++r) { const uint32_t i = w0 + r * 32 + lane; c[r] = i < a.n_claim ? __ldg(&a.claims[i]) : make_uint4(0, 0xFFFFFFFDu, 0, 0); }
    #pragma unroll
    for (int r = 0; r < 8; ++r) {
        const uint32_t i = w0 + r * 32 + lane, node = c[r].y;
        const bool stray = node >= a.n_node_global;
        const bool keep = i < a.n_claim && (stray ? a.take_stray != 0 : (node >= a.node_lo && node < a.node_hi));
        const uint32_t kind = c[r].x & 0xFFu, count = c[r].x >> 16;
        const uint32_t sl_any = i >= a.n_claim ? 0u : ((kind == DRA_KIND_GPU && !stray && !claim_invalid(kind, 0, count, a.have_off != 0)) ? count : 1u);
        const uint32_t sl = keep ? sl_any : 0u;
        if (a.world) {
            uint32_t o = 0;
            for (uint32_t q = 0; q + 1 < a.world; ++q) o += node >= a.rank_hi[q] ? 1u : 0u;
            own_sl[r] = ((stray ? a.stray_rank : o) << 16) | sl_any;
        }
        const uint32_t b = __ballot_sync(FULLMASK, keep);
        rk[r] = (uint32_t)__popc(b & ltm);
        keepm |= keep ? (1u << r) : 0u;
        const uint32_t ss = __reduce_add_sync(FULLMASK, sl);
        if (lane == 0) { rowc[wid * 8 + r] = (uint32_t)__popc(b); rows[wid * 8 + r] = ss; }
    }
    if (a.world) {                                           // slots per owner rank, for every rank (warp sums -> shared -> global)
        for (uint32_t q = 0; q < a.world; ++q) {
            uint32_t v = 0;
            #pragma unroll
            for (int r = 0; r < 8; ++r) v += (own_sl[r] >> 16) == q ? (own_sl[r] & 0xFFFFu) : 0u;
            v = __reduce_add_sync(FULLMASK, v);
            if (lane == 0 && v) atomicAdd(&rs_s[q], v);
        }
    }
    __syncthreads();
    if (a.world && tid < a.world && rs_s[tid]) atomicAdd(&a.rank_slots[(a.epoch & 1u) * PEER_MAX + tid], rs_s[tid]);
    if (wid == 0) {
        // exclusive scan of the 64 row counts (two per lane), tile totals
        const uint32_t c0 = rowc[2 * lane], c1 = rowc[2 * lane + 1], s0 = rows[2 * lane], s1 = rows[2 * lane + 1];
        uint32_t xc = c0 + c1, xs = s0 + s1;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t yc = __shfl_up_sync(FULLMASK, xc, d), ys = __shfl_up_sync(FULLMASK, xs, d);
            if (lane >= (uint32_t)d) { xc += yc; xs += ys; }
        }
        const uint32_t tc = __shfl_sync(FULLMASK, xc, 31), ts = __shfl_sync(FULLMASK, xs, 31);
        rowc[2 * lane] = xc - c0 - c1; rowc[2 * lane + 1] = xc - c1;
        // publish the aggregate, look back for the prefix, publish the inclusive prefix
        unsigned long long* st = a.status;
        if (lane == 0) atomicExch(&st[tile], sc_pack(a.epoch, tile == 0 ? 2u : 1u, tc, ts));
        uint32_t ec = 0, es = 0;
        int look = (int)tile - 1;
        const long long t0 = clock64();
        bool dead = false;
        while (look >= 0 && !dead) {
            const int idx = look - (int)lane;
            unsigned long long v = 0; bool ready;
            do {
                if (idx >= 0) asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(st + idx) : "memory");
                ready = idx < 0 || (((v >> 52) & 0x3FFu) == (a.epoch & 0x3FFu) && (v >> 62) != 0);
                if (clock64() - t0 > 2000000000ll) dead = true;
            } while (!__all_sync(FULLMASK, ready || dead));
            const uint32_t m2 = __ballot_sync(FULLMASK, idx < 0 || (v >> 62) == 2u);
            const uint32_t upto = m2 ? (uint32_t)__ffs(m2) - 1u : 31u;
            const bool inc = idx >= 0 && lane <= upto;
            ec += __reduce_add_sync(FULLMASK, inc ? (uint32_t)((v >> 26) & 0x3FFFFFFu) : 0u);
            es += __reduce_add_sync(FULLMASK, inc ? (uint32_t)(v & 0x3FFFFFFu) : 0u);
            if (m2) break;
            look -= 32;
        }
        if (dead && lane == 0) a.err.set(ERR_DEVICE_WAIT);
        if (lane == 0) {
            if (tile) atomicExch(&st[tile], sc_pack(a.epoch, 2u, ec + tc, es + ts));
            pre_c = ec; pre_s = es;
            if (tile == a.n_tiles - 1) {
                a.counts[0] = ec + tc; a.counts[1] = es + ts;
                a.h_counts[0] = ec + tc; a.h_counts[1] = es + ts; a.h_counts[3] = a.epoch;
                if (a.world) for (uint32_t q = 0; q < PEER_MAX; ++q) a.rank_slots[((a.epoch + 1u) & 1u) * PEER_MAX + q] = 0;   // the next call's counters
            }
        }
    }
    __syncthreads();
    const uint32_t base = pre_c;
    #pragma unroll
    for (int r = 0; r < 8; ++r) {
        if (!((keepm >> r) & 1u)) continue;
        const uint32_t i = w0 + r * 32 + lane;
        const uint32_t pos = base + rowc[wid * 8 + r] + rk[r];
        if (pos >= a.cap) { a.err.set(ERR_OUT_RANGE); continue; }
        uint4 v = c[r];
        v.y = v.y >= a.n_node_global ? 0xFFFFFFFFu : v.y - a.node_lo;
        a.cclaims[pos] = v;
        a.coff[pos] = a.out_off ? __ldg(&a.out_off[i]) : i;
    }
    if (a.timeline) { __syncthreads(); if (tid == 0) atomicMax(a.timeline + 1, globaltimer_ns()); }
}

// The same compaction for batches of up to 2M claims, built for LATENCY (the look-back form above walks a chain of
// dependent L2 round trips, a large share of the small batches it feeds).  Small tiles (ROWS x 256
// claims, all CTAs resident), and no chain at all: a tile publishes its aggregate and then reads the aggregates of
// ALL its predecessors at once (8 loads per lane in flight: 256 predecessors per L2 round trip), spinning only until the last of
// them has published.
// One tile (ROWS x 256 claims) by one CTA of 256 threads; used by the kernel below and, for shards that take the single-launch
// kernel, INSIDE k_fused (one tile per CTA, then a grid barrier: no second launch at all).
template <int ROWS>
__device__ __forceinline__ void shard_tile_flat(const ShardArgs& a, const uint32_t tile) {
    __shared__ uint32_t rowc[8 * ROWS], rows[8 * ROWS], pre_c, rs_s[PEER_MAX];
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, ltm = lanemask_lt();
    if (a.timeline && tid == 0) atomicMin(a.timeline, globaltimer_ns());
    if (tid < PEER_MAX) rs_s[tid] = 0;
    const uint32_t w0 = tile * (256 * ROWS) + wid * (32 * ROWS);
    uint4 c[ROWS]; uint32_t keepm = 0, own_sl[ROWS];
    #pragma unroll
    for (int r = 0; r < ROWS; ++r) { const uint32_t i = w0 + r * 32 + lane; c[r] = i < a.n_claim ? __ldg(&a.claims[i]) : make_uint4(0, 0xFFFFFFFDu, 0, 0); }
    __syncthreads();                                         // rs_s cleared
    #pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        const uint32_t i = w0 + r * 32 + lane, node = c[r].y;
        const bool stray = node >= a.n_node_global;
        const bool keep = i < a.n_claim && (stray ? a.take_stray != 0 : (node >= a.node_lo && node < a.node_hi));
        const uint32_t kind = c[r].x & 0xFFu, count = c[r].x >> 16;
        const uint32_t sl_any = i >= a.n_claim ? 0u : ((kind == DRA_KIND_GPU && !stray && !claim_invalid(kind, 0, count, a.have_off != 0)) ? count : 1u);
        uint32_t o = 0;
        for (uint32_t q = 0; q + 1 < a.world; ++q) o += node >= a.rank_hi[q] ? 1u : 0u;
        own_sl[r] = ((stray ? a.stray_rank : o) << 16) | sl_any;
        const uint32_t bm = __ballot_sync(FULLMASK, keep);
        keepm |= keep ? (1u << r) : 0u;
        const uint32_t ss = __reduce_add_sync(FULLMASK, keep ? sl_any : 0u);
        if (lane == 0) { rowc[wid * ROWS + r] = (uint32_t)__popc(bm); rows[wid * ROWS + r] = ss; }
    }
    for (uint32_t q = 0; q < a.world; ++q) {                  // slots per owner rank (for every rank: the gather's expected counts)
        uint32_t v = 0;
        #pragma unroll
        for (int r = 0; r < ROWS; ++r) v += (own_sl[r] >> 16) == q ? (own_sl[r] & 0xFFFFu) : 0u;
        v = __reduce_add_sync(FULLMASK, v);
        if (lane == 0 && v) atomicAdd(&rs_s[q], v);
    }
    __syncthreads();
    if (a.world && tid < a.world && rs_s[tid]) atomicAdd(&a.rank_slots[(a.epoch & 1u) * PEER_MAX + tid], rs_s[tid]);
    if (wid == 0) {
        // exclusive scan of the 8*ROWS row counts inside the tile (lane l holds rows l, l+32, ...)
        uint32_t tc = 0, ts = 0;
        constexpr int PER = (8 * ROWS + 31) / 32;
        uint32_t mc[PER], run = 0;
        #pragma unroll
        for (int k = 0; k < PER; ++k) { const uint32_t idx = lane * PER + k; mc[k] = idx < 8u * ROWS ? rowc[idx] : 0u; run += mc[k]; ts += idx < 8u * ROWS ? rows[idx] : 0u; }
        uint32_t x = run;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULLMASK, x, d); if (lane >= (uint32_t)d) x += y; }
        tc = __shfl_sync(FULLMASK, x, 31);
        ts = __reduce_add_sync(FULLMASK, ts);
        uint32_t ex = x - run;
        #pragma unroll
        for (int k = 0; k < PER; ++k) { const uint32_t idx = lane * PER + k; if (idx < 8u * ROWS) rowc[idx] = ex; ex += mc[k]; }
        // publish, then the prefix = sum of ALL predecessors' aggregates (every load in flight at once)
        unsigned long long* st = a.status;
        if (lane == 0) atomicExch(&st[tile], sc_pack(a.epoch, 1u, tc, ts));
        uint32_t ec = 0, es = 0;
        const long long t0 = clock64();
        bool dead = false;
        for (uint32_t base = 0; base < tile && !dead; base += 256) {
            unsigned long long v[8];
            bool ready;
            do {
                ready = true;
                #pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint32_t idx = base + k * 32 + lane;
                    v[k] = 0;
                    if (idx < tile) asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v[k]) : "l"(st + idx) : "memory");
                }
                #pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const uint32_t idx = base + k * 32 + lane;
                    if (idx < tile && !(((v[k] >> 52) & 0x3FFu) == (a.epoch & 0x3FFu) && (v[k] >> 62) != 0)) ready = false;
                }
                if (clock64() - t0 > 2000000000ll) dead = true;
            } while (!__all_sync(FULLMASK, ready || dead));
            #pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t idx = base + k * 32 + lane;
                if (idx < tile) { ec += (uint32_t)((v[k] >> 26) & 0x3FFFFFFu); es += (uint32_t)(v[k] & 0x3FFFFFFu); }
            }
        }
        ec = __reduce_add_sync(FULLMASK, ec); es = __reduce_add_sync(FULLMASK, es);
        if (dead && lane == 0) a.err.set(ERR_DEVICE_WAIT);
        if (lane == 0) {
            pre_c = ec;
            if (tile == a.n_tiles - 1) {
                a.counts[0] = ec + tc; a.counts[1] = es + ts;
                a.h_counts[0] = ec + tc; a.h_counts[1] = es + ts; a.h_counts[3] = a.epoch;
                if (a.world) for (uint32_t q = 0; q < PEER_MAX; ++q) a.rank_slots[((a.epoch + 1u) & 1u) * PEER_MAX + q] = 0;
            }
        }
    }
    __syncthreads();
    const uint32_t base = pre_c;
    #pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        // a lane's rank among the row's kept claims, from the keep mask again (fewer live registers than a stored rank)
        const uint32_t rk = (uint32_t)__popc(__ballot_sync(FULLMASK, (keepm >> r) & 1u) & ltm);
        if (!((keepm >> r) & 1u)) continue;
        const uint32_t i = w0 + r * 32 + lane;
        const uint32_t pos = base + rowc[wid * ROWS + r] + rk;
        if (pos >= a.cap) { a.err.set(ERR_OUT_RANGE); continue; }
        uint4 v = c[r];
        v.y = v.y >= a.n_node_global ? 0xFFFFFFFFu : v.y - a.node_lo;
        a.cclaims[pos] = v;
        a.coff[pos] = a.out_off ? __ldg(&a.out_off[i]) : i;
    }
    if (a.timeline) { __syncthreads(); if (tid == 0) atomicMax(a.timeline + 1, globaltimer_ns()); }
}

template <int ROWS>
__global__ void __launch_bounds__(256, 4)             // <= 64 registers: 4 CTAs per SM resident (528 on 132 SMs)
k_shard_compact_flat(const ShardArgs a) {
    pdl_trigger();
    shard_tile_flat<ROWS>(a, blockIdx.x);
}

// The flag-and-staging exchange of the sharded calls whose latency matters little (the rendezvous, UnsuitableNodes' bit
// exchange, the inventory sync): plain 16-byte stores into every peer's staging (k_peer_push), a system-scope fence, one
// flag per peer raised to the call's sequence number (peer_raise), and a bounded wait for every peer's flag here
// (peer_wait: ERR_PEER_TIMEOUT after spin_limit cycles, never a hang).  Monotonic sequence numbers: nothing is ever reset.
// Each exchange has its own region of the peer buffer; staging is double-buffered by call parity.
struct PeerExchange {
    uint4* stage[PEER_MAX];       // stage[p]: this rank's destination inside peer p's staging area (parity and slice applied)
    uint32_t* flag[PEER_MAX];     // flag[p]: this rank's flag word at peer p
    const uint4* my_stage;        // this rank's staging area (parity applied)
    const uint32_t* my_flags;     // [PEER_MAX], indexed by sender
    uint32_t world, rank, seq;
    long long spin_limit;         // clock cycles before a missing peer becomes ERR_PEER_TIMEOUT (never a hang)
    Err err;
};

// thread tid raises this rank's flag at peer tid, after a system-scope fence: the staged stores before it are seen first
__device__ __forceinline__ void peer_raise(const PeerExchange& x, uint32_t tid) {
    if (tid >= x.world || tid == x.rank) return;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(x.flag[tid]), "r"(x.seq) : "memory");
}
// thread tid waits until peer tid's flag here has reached the call's sequence number; false (ERR_PEER_TIMEOUT set) once
// spin_limit cycles have passed since t0
__device__ __forceinline__ bool peer_wait(const PeerExchange& x, uint32_t tid, long long t0) {
    if (tid >= x.world || tid == x.rank) return true;
    uint32_t v;
    do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(x.my_flags + tid) : "memory");
        if ((int32_t)(v - x.seq) >= 0) return true;
    } while (clock64() - t0 <= x.spin_limit);
    x.err.set(ERR_PEER_TIMEOUT);
    return false;
}

// src[lo, hi) into stage[p] at the same indices for every peer p, then a system-scope fence per thread.  Nothing waits here.
__global__ void __launch_bounds__(256)
k_peer_push(const PeerExchange x, const uint4* __restrict__ src, uint32_t lo, uint32_t hi) {
    for (uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) {
        const uint4 v = __ldcg(&src[i]);
        for (uint32_t p = 0; p < x.world; ++p)
            if (p != x.rank) x.stage[p][i] = v;
    }
    __threadfence_system();
}

// Cross-rank rendezvous on the device (dra_peer_rendezvous_device): the exchange's flags alone, nothing staged.  Orders
// nothing but time — it lines the ranks' streams up (a benchmark uses it after its untimed L2 flush so that a rank's timed
// step does not absorb its peers' flush-duration skew).
__global__ void __launch_bounds__(32)
k_rendezvous(const PeerExchange x) {
    peer_raise(x, threadIdx.x);
    peer_wait(x, threadIdx.x, clock64());
}

// ====================================================================================================
// pack: first-fit per node
// ====================================================================================================

// ---- the path's one collective: all-gather of OutRecs as self-validating 16-byte packets over NVLink ----------------
// A flag round trip between two GPUs costs microseconds, a system fence after remote stores costs a full round trip,
// and tens of thousands of scattered 8-byte remote stores take longer still to drain (profiles/peer_bench.cu measures
// each).  So: no fence, no flag, no ticket.  Every OutRec travels as ONE 16-byte store
//   { gpu, meta | tag(epoch) in meta's spare bits, table slot, epoch }
// into a staging slice of the receiver (each 8-byte half carries its own validity tag, so even a torn read is
// caught); a CTA reserves a CONTIGUOUS range of its rank's slice with one atomicAdd, so a node's ~80 packets leave as
// ~10 full 128-byte lines instead of 80 sector writes — the slot rides in the packet, order does not matter.
// Receivers poll their own (local) staging memory and scatter the records into the result table.  Latency after the
// slowest CTA of any rank: one NVLink hop + one L2 probe.
constexpr uint32_t PKT_CLEAN = ~(0xF0u | 0xE000u | 0xF8000000u);      // meta bits that are always zero (start <= 15, size <= 16, status <= 7)
struct PktGather {
    uint4* stage[PEER_MAX];       // stage[p]: THIS rank's slice inside peer p's staging area (parity applied)
    uint4* hdr[PEER_MAX];         // hdr[p]: this rank's header slot at peer p
    const uint4* my_stage;        // this rank's own staging area: slice r at my_stage + r * cap
    const uint4* my_hdr;          // [world]
    uint2* table;                 // this rank's result table (parity applied)
    uint32_t* cursor;             // [2] reservation cursors, one per parity
    uint32_t world, rank, cap, epoch, parity;
    uint32_t slot_base;           // table index of this rank's local slot 0 (slice form: rank * n_per; global form: 0)
    uint32_t n_per;               // slice form: every rank's padding [count_r, n_per) is zeroed by the receiver; 0: global slots
    uint32_t count;               // packets (OutRec slots) this rank sends, when the host knows it ...
    const uint32_t* count_dev;    // ... else it is read here
    long long spin_limit;         // clock cycles before a missing packet becomes ERR_PEER_TIMEOUT (never a hang)
    const uint32_t* expect;       // [world] packets every rank will send, known BEFORE the kernel starts (sharded call: every
                                  // rank reads the whole claim array and counts all ranks' slots) — then no header is waited for
};

__device__ __forceinline__ uint32_t pkt_tag(uint32_t meta, uint32_t epoch) {
    const uint32_t t = epoch & 0xFFFu;
    return meta | ((t & 0xFu) << 4) | (((t >> 4) & 7u) << 13) | (((t >> 7) & 0x1Fu) << 27);
}
__device__ __forceinline__ void pkt_store(uint4* p, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ uint4 pkt_load(const uint4* p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
// header of this rank to every peer: how many packets it has sent (0xFFFFFFFF: it gave up).  One thread per peer.
// Sent by the LAST sending CTA with the final value of the reservation cursor, so the count is exactly what went out
// even when the caller's out_off leaves gaps.
__device__ __forceinline__ void pkt_send_header(const PktGather& g, uint32_t p, uint32_t n) {
    if (p >= g.world || p == g.rank) return;
    pkt_store(g.hdr[p], n, n ^ g.epoch ^ 0xA5A5A5A5u, 0u, g.epoch);
}
// CTA-collective: called by every CTA of the grid once its packets are out; the last one publishes the count
__device__ __forceinline__ void pkt_finish_send(const PktGather& g) {
    __shared__ uint32_t last_s, total_s;
    if (g.expect) return;                              // the receivers already know the counts: no ticket, no header
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const bool last = atomicAdd(&g.cursor[2u + g.parity], 1u) == gridDim.x - 1;
        if (last) { g.cursor[2u + g.parity] = 0; total_s = atomicAdd(&g.cursor[g.parity], 0u); }
        last_s = last ? 1u : 0u;
    }
    __syncthreads();
    if (last_s) {
        pkt_send_header(g, threadIdx.x, total_s);
        // slice form: the padding of this rank's own slice (the peers zero their copies of it when the header arrives)
        if (g.n_per) for (uint32_t k = total_s + threadIdx.x; k < g.n_per; k += blockDim.x) g.table[g.slot_base + k] = make_uint2(0u, 0u);
    }
}
// one record to every peer at position pos of this rank's slice
__device__ __forceinline__ void pkt_send(const PktGather& g, uint32_t pos, uint2 rec, uint32_t slot) {
    const uint32_t y = pkt_tag(rec.y, g.epoch);
    #pragma unroll 1
    for (uint32_t p = 0; p < g.world; ++p)
        if (p != g.rank) pkt_store(g.stage[p] + pos, rec.x, y, slot, g.epoch);
}
// Receive side, thread T of NT: poll the local staging slices until every peer's packets are in, scatter into the table.
// A position is done when its packet is valid, or when the peer's header says nothing will come there.
__device__ __forceinline__ void pkt_receive(const PktGather& g, uint32_t T, uint32_t NT, const Err& err) {
    if (g.expect) {
        // Counts known up front: the packets of ALL peers form one work list; a thread's items are loaded together (one L2
        // round trip for all of them, whichever peer they come from) and only the ones not yet in are asked for again.
        // (Walking peer after peer costs one dependent round trip per peer even when everything has already arrived.)
        const uint32_t want_tag = pkt_tag(0u, g.epoch);
        const long long t0 = clock64();
        uint32_t total = 0;
        for (uint32_t r = 0; r < g.world; ++r) if (r != g.rank) total += min(__ldcg(g.expect + r), g.cap);
        auto locate = [&](uint32_t j) -> const uint4* {               // item j of the concatenated slices
            for (uint32_t r = 0; r < g.world; ++r) {
                if (r == g.rank) continue;
                const uint32_t n = min(__ldcg(g.expect + r), g.cap);
                if (j < n) return g.my_stage + (size_t)r * g.cap + j;
                j -= n;
            }
            return g.my_stage;
        };
        constexpr int MAXI = 4;
        bool dead = false;
        for (uint32_t b0 = T; b0 < total && !dead; b0 += NT * MAXI) {
            const uint4* p[MAXI]; uint32_t pend = 0;
            #pragma unroll
            for (int i = 0; i < MAXI; ++i) { const uint32_t j = b0 + (uint32_t)i * NT; p[i] = locate(j < total ? j : 0u); if (j < total) pend |= 1u << i; }
            uint32_t spins = 0;
            while (pend && !dead) {
                uint4 v[MAXI];
                #pragma unroll
                for (int i = 0; i < MAXI; ++i) if ((pend >> i) & 1u) v[i] = pkt_load(p[i]);
                #pragma unroll
                for (int i = 0; i < MAXI; ++i)
                    if (((pend >> i) & 1u) && v[i].w == g.epoch && (v[i].y & ~PKT_CLEAN) == want_tag) {
                        g.table[v[i].z] = make_uint2(v[i].x, v[i].y & PKT_CLEAN);
                        pend &= ~(1u << i);
                    }
                if (pend && (++spins & 63u) == 0) {
                    if (clock64() - t0 > g.spin_limit) dead = true;
                    if ((spins & 1023u) == 0)                          // a peer that gave up says so in its header
                        for (uint32_t r = 0; r < g.world; ++r) {
                            if (r == g.rank) continue;
                            const uint4 h = pkt_load(g.my_hdr + r);
                            if (h.w == g.epoch && h.x == 0xFFFFFFFFu && h.y == (h.x ^ g.epoch ^ 0xA5A5A5A5u)) dead = true;
                        }
                }
            }
        }
        if (dead) err.set(ERR_PEER_TIMEOUT);
        return;
    }
    const uint32_t want_tag = pkt_tag(0u, g.epoch);
    const long long t0 = clock64();
    bool dead = false;
    for (uint32_t r = 0; r < g.world && !dead; ++r) {
        if (r == g.rank) continue;                                    // own records went straight into the table
        uint32_t n = g.expect ? min(__ldcg(g.expect + r), g.cap) : 0xFFFFFFFFu;     // unknown until the header is in
        const uint4* sl = g.my_stage + (size_t)r * g.cap;
        uint32_t spins = 0;
        for (uint32_t k = T; !dead; ) {
            if (n == 0xFFFFFFFFu) {
                const uint4 h = pkt_load(g.my_hdr + r);
                if (h.w == g.epoch && h.y == (h.x ^ g.epoch ^ 0xA5A5A5A5u)) {
                    if (h.x == 0xFFFFFFFFu) { dead = true; break; }    // the peer aborted its batch
                    n = min(h.x, g.cap);
                }
            }
            if (n != 0xFFFFFFFFu && k >= n) break;
            if (k < g.cap) {
                const uint4 v = pkt_load(sl + k);
                if (v.w == g.epoch && (v.y & ~PKT_CLEAN) == want_tag) {
                    g.table[v.z] = make_uint2(v.x, v.y & PKT_CLEAN);
                    k += NT; spins = 0;
                    continue;
                }
            }
            if ((++spins & 63u) == 0) {
                if (clock64() - t0 > g.spin_limit) dead = true;
                if (g.expect && (spins & 1023u) == 0) {              // a peer that gave up says so in its header
                    const uint4 h = pkt_load(g.my_hdr + r);
                    if (h.w == g.epoch && h.x == 0xFFFFFFFFu && h.y == (h.x ^ g.epoch ^ 0xA5A5A5A5u)) dead = true;
                }
            }
        }
        if (g.n_per && !dead) for (uint32_t k = n + T; k < g.n_per; k += NT) g.table[(size_t)r * g.n_per + k] = make_uint2(0u, 0u);
    }
    if (dead) err.set(ERR_PEER_TIMEOUT);
}

// Direct host I/O of the single-launch kernel (k_fused): the CTAs themselves ingest the batch from the caller's
// pinned (device-mapped) host buffers and write the OutRecs back there, instead of copy-engine transfers around the
// kernel.  Needs every CTA resident at once (cooperative launch): two grid-wide barriers.
struct DirectIO {
    const uint4* h_claims;        // NULL: off
    const uint32_t* h_out_off;    // or NULL
    uint2* h_out;
    uint4* d_claims;              // device copies the kernel body reads (= PackArgs::claims / out_off)
    uint32_t* d_out_off;
    uint32_t* gbar;               // [0] arrival count, [1] generation (self-resetting, reusable across launches)
};

struct PackArgs {
    const uint4* sorted;          // node-sorted claims, .y = first out slot          (k_pack)
    const uint32_t* claim_off;    // [n_node+2]                                        (k_pack)
    const uint4* claims;          // claims in input order                             (k_fused)
    const uint32_t* out_off;      // first out slot per claim or NULL                  (k_fused)
    uint32_t n_claim;             //                                                   (k_fused)
    ShardArgs sh; uint32_t sh_on; // sharded call, shard small enough: the compaction runs INSIDE this kernel (one tile per CTA)  (k_fused)
    uint32_t q_cap;               // multi-GPU: entries of the shared-memory send queue behind the staged claims (0: none) (k_fused)
    const uint32_t* n_dev;        // if set: the real number of claims (<= n_claim, which then only sizes the layout) (k_fused)
    const uint4* inv_src;         // inventory read from here ...
    uint4* inv_dst;               // ... and written back here (may alias inv_src)
    const uint32_t* node_off;     // [n_node+1]
    const uint32_t* tbl;          // [16*16] ProfEnt as u32
    uint2* out;
    uint32_t n_out, n_node, have_off;
    Err err;
    SelCtx sel;                   // optional GPU attributes + selector table (spec §10)
    PktGather peer;               // world == 0: single GPU                            (k_fused)
    unsigned long long* timeline; // optional instrumentation: 8 clock stamps per CTA  (k_fused), else NULL
    DirectIO dio;                 //                                                   (k_fused)
};

__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lop3_or(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d; asm("lop3.b32 %0, %1, %2, %3, 0xFE;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
__device__ __forceinline__ uint32_t lop3_nor(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d; asm("lop3.b32 %0, %1, %2, %3, 0x01;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d;
}
__device__ __forceinline__ void sts32_if(bool p, uint32_t addr, uint32_t v) {     // predicated, no branch
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p st.shared.u32 [%0], %1;\n\t}" ::"r"(addr), "r"(v), "r"((uint32_t)p) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void mbar_init_a(uint32_t addr, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(addr), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_inval_a(uint32_t addr) {
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t addr, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    } while (!ok);
}
// 1-D TMA bulk copy global -> shared (shared-space addresses), completion on an mbarrier
__device__ __forceinline__ void tma_load_a(uint32_t sdst, const void* gsrc, uint32_t bytes, uint32_t bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(bar) : "memory");
}
// shared-space base of the dynamic shared memory, made opaque so that it lives in a register instead of
// being rematerialised from SR_CgaCtaId at every use
__device__ __forceinline__ uint32_t smem_base(const void* dyn) {
    uint32_t b = smem_u32(dyn);
    asm volatile("" : "+r"(b));
    return b;
}

// shift schedule of fit_map for a given size, 4 nibbles: t &= t >> s_i, i = 0..3 (covers sizes 1..16)
__device__ __forceinline__ uint32_t shifts_of(uint32_t size) {
    uint32_t c = 1, sh = 0;
    #pragma unroll
    for (int i = 0; i < 4; ++i) { const uint32_t s_ = min(c, size - c) & 15u; sh |= s_ << (4 * i); c += s_; }
    return sh;
}

// The warp that packs one node: one lane per GPU.
struct NodeCtx {
    Lane L; Dead D; OutSink sink;
    uint32_t lane, ltmask, g0, m0, k_next;
    uint32_t gate;                 // 0xFFFF on lanes whose GPU can take MIG devices at all, else 0
    bool small8;                   // homogeneous node whose table row has no shape larger than 8 slices
    bool offer_any;                // some GPU of the node is MIG-enabled and available (offers its table row)
    uint32_t live_addr;            // shared: 32 prepared records x 32 B, followed by 32 result words
    uint32_t tbl_addr;             // shared: placement table (u32 cells)
    const uint32_t* tbl_ptr;       // same table for the generic step
    bool homog, mig_ok, mig_offer, have_off;
    SelCtx sc;
    bool prof_on = false;          // instrumentation: cycle accumulators of the three parts of segment_run
    long long t_pre = 0, t_loop = 0, t_epi = 0, t_pre_a = 0, t_fetch = 0; uint32_t n_live = 0;

    __device__ __forceinline__ void begin(uint4 rec, bool valid) {
        constexpr uint32_t BLOCKED = DRA_GPU_MIG_ENABLED | DRA_GPU_FULL_ALLOCATED | DRA_GPU_UNAVAILABLE;
        L.load(rec, valid);
        D = Dead();
        k_next = 0;
        // facts that cannot change during the batch (FULL is only ever set on non-MIG GPUs)
        mig_offer = L.valid && (L.flags & (DRA_GPU_MIG_ENABLED | DRA_GPU_UNAVAILABLE)) == DRA_GPU_MIG_ENABLED;
        mig_ok = L.valid && (L.flags & BLOCKED) == DRA_GPU_MIG_ENABLED;
        gate = mig_ok ? 0xFFFFu : 0u;
        m0 = __shfl_sync(FULLMASK, L.model, 0);
        homog = __all_sync(FULLMASK, !L.valid || L.model == m0);     // one placement-table row for the node
        offer_any = __any_sync(FULLMASK, mig_offer);
        small8 = homog && __all_sync(FULLMASK, lane >= DRA_MAX_PROFILES ||
                                     (lds32(tbl_addr + ((m0 * DRA_MAX_PROFILES + (lane & (DRA_MAX_PROFILES - 1))) << 2)) & 0xFFu) <= 8u);
    }
};

// One segment of <= 32 consecutive claims of the node; lane j holds claim j (c.y = first out slot).
//   1. lane-parallel: malformed claims and request shapes already known to fail on this node (Dead memo)
//      write their own OutRec, 32 at a time; live claims are compacted, in order, into prepared records;
//   2. serial: the live records, in order — candidate starts by a log-step shift/AND on the lane's occupancy
//      mask, __ballot_sync + __ffs = lowest GPU, __ffs of the winner's candidates = lowest start.
template <class Get>
__device__ __forceinline__ void segment_run(NodeCtx& x, const uint4 c, const bool present, const uint32_t pos,
                                            Get get, const uint32_t cnt) {
    constexpr uint32_t BLOCKED = DRA_GPU_MIG_ENABLED | DRA_GPU_FULL_ALLOCATED | DRA_GPU_UNAVAILABLE;
    Lane& L = x.L; Dead& D = x.D; OutSink& sink = x.sink;
    const uint32_t lane = x.lane, g0 = x.g0;
    long long tq0 = 0; if (x.prof_on) tq0 = clock64();
    const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
    const uint32_t dst = c.y, mem = c.z, group = c.w;
    // Straight-line and predicated: nested divergent regions cost this warp more than the arithmetic they skip
    // (profiles/timeline.py shows it).  The rare paths (range error, multi-slot emission) sit behind votes.
    bool live = present && pos >= x.k_next;
    const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : prof;
    const uint32_t sel = claim_sel(kind, mem, group);
    const bool inval = claim_invalid(kind, prof, count, x.have_off);       // spec §3 (unknown selector ids: generic step)
    const uint32_t slots = (kind == DRA_KIND_GPU && !inval) ? count : 1u;
    // co-location runs and claims with a selector take the generic step (own range checks, no failure memo)
    const bool is_group = !inval && ((kind == DRA_KIND_MIG && group != 0) || sel != 0);
    const bool oor = live && !is_group && (inval ? dst >= sink.n_out : (dst > sink.n_out || slots > sink.n_out - dst));
    uint32_t st = inval ? (uint32_t)DRA_ST_INVALID : 0xFFu;                // 0xFF: nothing to emit, the claim stays live
    {                                                                      // shapes that already failed here
        const uint32_t pbit = 1u << (prof & 31u);
        const bool mig = kind == DRA_KIND_MIG, gpu = kind == DRA_KIND_GPU;
        const bool dead = mig ? ((D.bad | D.nocap) & pbit) != 0 : gpu ? count >= D.gpu_min : (uint64_t)mem >= D.sh_min;
        const uint32_t dst_ = mig ? ((D.bad & pbit) ? DRA_ST_BAD_PROFILE : DRA_ST_NO_CAPACITY) : gpu ? DRA_ST_NO_CAPACITY : DRA_ST_MEM_LIMIT;
        st = (!inval && !is_group && dead) ? dst_ : st;
    }
    const bool emit = live && !oor && st != 0xFFu;
    if (emit && slots == 1u) sink.put(dst, DRA_GPU_NONE, meta(0, 0, op, st));
    if (__any_sync(FULLMASK, oor || (emit && slots != 1u))) {              // rare
        if (oor) sink.err.set(ERR_OUT_RANGE);
        if (emit && slots != 1u) for (uint32_t s_ = 0; s_ < slots; ++s_) sink.put(dst + s_, DRA_GPU_NONE, meta(0, 0, op, st));
    }
    live = live && !oor && st == 0xFFu;
    if (x.prof_on) x.t_pre_a += clock64() - tq0;           // validity / range / dead-shape part of the pre-pass
    // prepared record of a live claim (what the serial step needs, already unpacked):
    //   r0 = {s1, s2, s3, s4}  shift schedule (MIG) | {count or mem or position, 0, 0, 0}
    //   r1 = {smask | prof<<16 | class<<24, first out slot, OutRec meta (size<<8 | prof<<16), (1<<size)-1}
    const uint32_t lm = __ballot_sync(FULLMASK, live);
    if (lm == 0) return;
    if (live) {
        uint4 r0 = make_uint4(0, 0, 0, 0), r1 = make_uint4(0, dst, 0, 0);
        uint32_t fail_word = 0;
        if (is_group) { r0.x = pos; r1.x = 4u << 24; }
        else if (kind == DRA_KIND_MIG) {
            const uint32_t e = lds32(x.tbl_addr + ((x.m0 * DRA_MAX_PROFILES + prof) << 2));   // homogeneous node: one cell for all GPUs
            const uint32_t size = e & 0xFFu, sh = shifts_of(size);
            r0 = make_uint4(sh & 15u, (sh >> 4) & 15u, (sh >> 8) & 15u, sh >> 12);
            r1.x = (e >> 16) | (prof << 16) | (1u << 24);
            r1.z = (size << 8) | (prof << 16);
            r1.w = (1u << size) - 1u;
            // the record's result word starts out as its failure: static on a homogeneous node (the row offers the
            // shape or it does not); the lean loop only overwrites it on success
            fail_word = 0xFFu | (((x.offer_any && (e >> 16) != 0) ? DRA_ST_NO_CAPACITY : DRA_ST_BAD_PROFILE) << 24);
        } else if (kind == DRA_KIND_GPU) { r0.x = count; r1.x = 2u << 24; }
        else { r0.x = mem; r1.x = 3u << 24; fail_word = 0xFFu | (DRA_ST_MEM_LIMIT << 24); }
        const uint32_t qi = (uint32_t)__popc(lm & x.ltmask);
        const uint32_t at = x.live_addr + (qi << 5);
        sts128(at, r0); sts128(at + 16, r1);
        sts32(x.live_addr + 1024 + (qi << 2), fail_word);
    }
    __syncwarp();
    const uint32_t nlive = (uint32_t)__popc(lm);
    long long tq1 = 0; if (x.prof_on) { tq1 = clock64(); x.t_pre += tq1 - tq0; x.n_live += nlive; }

    // One live record: mutates L / D.  MIG and SHARED steps only RECORD their outcome in shared memory
    // (res[q] = winner lane | start<<8 | size<<16, or 0xFF | status<<24); the OutRecs are composed and stored
    // after the loop, 32 at a time — nothing but the first-fit chain itself stays on the serial path.
    const uint32_t res_addr = x.live_addr + 1024;
    auto step = [&](const uint4 r0, const uint4 r1, const uint32_t q) {
        const uint32_t cls = r1.x >> 24, dj = r1.y;
        if (cls == 1u) {                                   // MIG, spec §5
            const uint32_t pj = (r1.x >> 16) & 0xFFu;
            if (((D.bad | D.nocap) >> pj) & 1u) {          // shape died earlier in this segment
                if (lane == 0) sts32(res_addr + (q << 2), 0xFFu | ((((D.bad >> pj) & 1u) ? DRA_ST_BAD_PROFILE : DRA_ST_NO_CAPACITY) << 24));
                return;
            }
            uint32_t smask = r1.x & 0xFFFFu, s1 = r0.x, s2 = r0.y, s3 = r0.z, s4 = r0.w, sbits = r1.w, size = (r1.z >> 8) & 0xFFu;
            if (!x.homog) {                                // per-GPU table row
                const uint32_t e = lds32(x.tbl_addr + ((L.model * DRA_MAX_PROFILES + pj) << 2));
                const uint32_t sh = shifts_of(e & 0xFFu);
                size = e & 0xFFu; smask = e >> 16; s1 = sh & 15u; s2 = (sh >> 4) & 15u; s3 = (sh >> 8) & 15u; s4 = sh >> 12;
                sbits = (1u << size) - 1u;
            }
            uint32_t t = ~L.busy & x.gate;
            t &= t >> s1; t &= t >> s2; t &= t >> s3; t &= t >> s4;
            const uint32_t cand = t & smask;
            const uint32_t b = __ballot_sync(FULLMASK, cand != 0);
            const uint32_t st = (uint32_t)__ffs(cand) - 1u;              // lowest start (if this lane wins)
            const bool win = lane == (uint32_t)__ffs(b) - 1u;            // lowest GPU; b == 0: nobody
            if (win) { L.busy |= sbits << (st & 31u); sts32(res_addr + (q << 2), lane | (st << 8) | (size << 16)); }
            if (b == 0) {
                const bool any = __ballot_sync(FULLMASK, x.mig_offer && smask != 0) != 0;
                if (any) D.nocap |= 1u << pj; else D.bad |= 1u << pj;
                if (lane == 0) sts32(res_addr + (q << 2), 0xFFu | ((any ? DRA_ST_NO_CAPACITY : DRA_ST_BAD_PROFILE) << 24));
            }
        } else if (cls == 2u) {                            // full GPUs, spec §4 (several slots: emitted here)
            const uint32_t cj = r0.x;
            if (cj >= D.gpu_min) { if (lane < cj) sink.put(dj + lane, DRA_GPU_NONE, meta(0, 0, DRA_PROFILE_GPU, DRA_ST_NO_CAPACITY)); return; }
            const bool elig = L.valid && !(L.flags & BLOCKED) && L.share == 0;
            const uint32_t b = __ballot_sync(FULLMASK, elig);
            const uint32_t r = (uint32_t)__popc(b & x.ltmask);
            if ((uint32_t)__popc(b) >= cj) {
                if (elig && r < cj) { L.flags |= DRA_GPU_FULL_ALLOCATED; sink.put(dj + r, g0 + lane, meta(0, 0, DRA_PROFILE_GPU, DRA_ST_OK)); }
            } else {
                D.gpu_min = cj;
                if (lane < cj) sink.put(dj + lane, DRA_GPU_NONE, meta(0, 0, DRA_PROFILE_GPU, DRA_ST_NO_CAPACITY));
            }
        } else if (cls == 3u) {                            // shared GPU, spec §7
            const uint32_t mj = r0.x;
            if ((uint64_t)mj >= D.sh_min) { if (lane == 0) sts32(res_addr + (q << 2), 0xFFu | (DRA_ST_MEM_LIMIT << 24)); return; }
            const bool elig = L.valid && !(L.flags & BLOCKED) && L.share < 0xFFFFu && L.mem >= mj;
            const uint32_t b = __ballot_sync(FULLMASK, elig);
            const bool win = lane == (uint32_t)__ffs(b) - 1u;
            if (win) { L.mem -= mj; L.share += 1; sts32(res_addr + (q << 2), lane); }
            if (b == 0) {
                D.sh_min = mj;
                if (lane == 0) sts32(res_addr + (q << 2), 0xFFu | (DRA_ST_MEM_LIMIT << 24));
            }
        } else {                                           // co-location run: generic step (emits its own records)
            const uint32_t pj = r0.x;
            if (pj >= x.k_next) {
                // by COPY: the out-of-line call takes references, and a reference into the node context would
                // pin the whole context (lane state, memo, sink) in local memory — every access an LDL
                Lane Lt = L; Dead Dt = D; auto St = sink;
                const uint32_t used = node_step_cold(Lt, Dt, lane, g0, x.tbl_ptr, get, pj, cnt, St, x.have_off, x.sc);
                L = Lt; D = Dt; sink = St;
                x.k_next = pj + used;
            }
        }
    };
    // Common case — every live record of the segment is a plain MIG claim on a homogeneous node: a loop with
    // no class dispatch and no divergent branch.  Winner = lowest set bit of the ballot (b & -b, no FLO on the
    // chain), placement bits = sizebits * lowest-candidate-bit (a multiply by a one-hot is the shift).
    const bool fast = x.homog && __ballot_sync(FULLMASK, live && (is_group || kind != DRA_KIND_MIG)) == 0;
    const bool fast_sh = !fast && __ballot_sync(FULLMASK, live && (is_group || kind != DRA_KIND_SHARED)) == 0;
    const uint32_t lanebit = 1u << lane;
    if (fast_sh) {
        // every live record is a SHARED claim (spec §7): flags cannot change inside the segment
        const bool share_ok = L.valid && !(L.flags & BLOCKED);
        // lean, like the MIG loop below: the memo is not read (a limit at or above one that failed finds no GPU:
        // free memory only shrinks), failures are the pre-initialised result words, memo update in the epilogue
        const uint32_t lemask = lanebit | (lanebit - 1u);
        auto sstep = [&](const uint4 r0, const uint32_t q) {
            const uint32_t mj = r0.x;
            const bool elig = share_ok && L.share < 0xFFFFu && L.mem >= mj;
            const uint32_t b = __ballot_sync(FULLMASK, elig);
            const bool lose = ((b & lemask) ^ lanebit) != 0;               // win: lowest eligible GPU
            L.mem = lose ? L.mem : L.mem - mj; L.share += lose ? 0u : 1u;
            sts32_if(!lose, res_addr + (q << 2), lane);
        };
        uint4 a0 = lds128(x.live_addr), b0;
        for (uint32_t q = 0; q < nlive; q += 2) {
            const uint32_t nb_ = x.live_addr + ((q + 1) << 5);
            if (q + 1 < nlive) b0 = lds128(nb_);
            sstep(a0, q);
            if (q + 1 >= nlive) break;
            if (q + 2 < nlive) a0 = lds128(nb_ + 32);
            sstep(b0, q + 1);
        }
    } else if (fast) {
        // Lean step (profiles/chain_bench.cu measures it against the earlier forms).  A single warp is
        // bound by max(loop-carried chain at ~6 cycles per dependent ALU op, 2 cycles per ALU instruction), so:
        //  - the state is the FREE mask (no NOT on the chain), 0 on lanes that cannot take MIG devices;
        //  - the start mask is static: a shape that died earlier simply finds no candidate (occupancy only grows), so
        //    the dead-shape memo is not read here; it is brought up to date once, in the epilogue;
        //  - no failure handling at all: the pre-pass initialised every result word to the shape's (static) failure;
        //  - winner test = one LOP3 with a predicate output, update = select between two precomputed masks.
        uint32_t fre = ~L.busy & x.gate;
        const uint32_t lemask = lanebit | (lanebit - 1u), gate = x.gate;
        auto fstep = [&](auto NRtag, const uint4 r0, const uint4 r1, const uint32_t q) {
            uint32_t t = fre;
            t &= t >> r0.x; t &= t >> r0.y; t &= t >> r0.z;
            if (decltype(NRtag)::value == 4) t &= t >> r0.w;               // shapes of 9..16 slices
            const uint32_t cand = t & r1.x & gate;                         // gate has 16 bits: drops prof/class of r1.x
            const uint32_t b = __ballot_sync(FULLMASK, cand != 0);
            const uint32_t low = cand & (0u - cand);                       // lowest start, one-hot
            const uint32_t freW = fre & ~(r1.w * low);                     // off the chain: overlaps the vote
            const bool lose = ((b & lemask) ^ lanebit) != 0;               // win: lowest GPU with a candidate
            fre = lose ? fre : freW;
            sts32_if(!lose, res_addr + (q << 2), lane + (cand << 8));      // start = lowest set bit, decoded in the epilogue
        };
        auto floop = [&](auto NRtag) {
            uint4 a0 = lds128(x.live_addr), a1 = lds128(x.live_addr + 16), b0, b1;
            for (uint32_t q = 0; q < nlive; q += 2) {
                const uint32_t nb_ = x.live_addr + ((q + 1) << 5);
                if (q + 1 < nlive) { b0 = lds128(nb_); b1 = lds128(nb_ + 16); }
                fstep(NRtag, a0, a1, q);
                if (q + 1 >= nlive) break;
                if (q + 2 < nlive) { a0 = lds128(nb_ + 32); a1 = lds128(nb_ + 48); }
                fstep(NRtag, b0, b1, q + 1);
            }
        };
        if (x.small8) floop(std::integral_constant<int, 3>{}); else floop(std::integral_constant<int, 4>{});
        L.busy = gate ? (~fre & 0xFFFFu) : L.busy;
    } else {
    // ping-pong: the next record is in flight while the current one is stepped, no register shuffling
    uint4 a0 = lds128(x.live_addr), a1 = lds128(x.live_addr + 16), b0, b1;
    for (uint32_t q = 0; q < nlive; q += 2) {
        const uint32_t nb_ = x.live_addr + ((q + 1) << 5);
        if (q + 1 < nlive) { b0 = lds128(nb_); b1 = lds128(nb_ + 16); }
        step(a0, a1, q);
        if (q + 1 >= nlive) break;
        if (q + 2 < nlive) { a0 = lds128(nb_ + 32); a1 = lds128(nb_ + 48); }
        step(b0, b1, q + 1);
    }
    }
    __syncwarp();
    long long tq2 = 0; if (x.prof_on) { tq2 = clock64(); x.t_loop += tq2 - tq1; }
    // epilogue: lane q composes and stores the OutRec of live record q (MIG / SHARED)
    uint32_t died_nocap = 0, died_bad = 0;                 // lean loop: shapes that failed in this segment
    {
        // predicated straight-line code (one store), not nested branches
        const bool have = lane < nlive;
        uint4 r1 = make_uint4(0, 0, 0, 0); uint32_t res = 0;
        if (have) { r1 = lds128(x.live_addr + (lane << 5) + 16); res = lds32(res_addr + (lane << 2)); }
        const uint32_t cls = r1.x >> 24;
        const bool mine = have && (cls == 1u || cls == 3u);
        const uint32_t w = res & 0xFFu, st_ = res >> 24;
        const uint32_t prof_ = cls == 1u ? ((r1.x >> 16) & 0xFFu) : (uint32_t)DRA_PROFILE_SHARED;
        const bool failed = w == 0xFFu;
        const uint32_t pbit = 1u << (prof_ & 31u);
        died_nocap = (fast && mine && failed && st_ == DRA_ST_NO_CAPACITY) ? pbit : 0u;
        died_bad = (fast && mine && failed && st_ != DRA_ST_NO_CAPACITY) ? pbit : 0u;
        const uint32_t m_ok = fast ? (r1.z | ((uint32_t)__ffs((res >> 8) & 0xFFFFu) - 1u))
                                   : meta((res >> 8) & 0xFFu, (res >> 16) & 0xFFu, prof_, DRA_ST_OK);
        const uint32_t gpu_ = failed ? (uint32_t)DRA_GPU_NONE : g0 + w;
        const uint32_t m_ = failed ? meta(0, 0, prof_, st_) : m_ok;
        if (mine) sink.put(r1.y, gpu_, m_);
        if (fast_sh) {                                     // smallest limit that failed in this segment
            const uint32_t fm = (mine && failed) ? lds32(x.live_addr + (lane << 5)) : 0xFFFFFFFFu;
            const uint32_t mn = __reduce_min_sync(FULLMASK, fm);
            if ((uint64_t)mn < D.sh_min && mn != 0xFFFFFFFFu) D.sh_min = mn;
        }
    }
    if (fast) {                                            // the dead-shape memo, for the next segment's pre-pass
        D.nocap |= __reduce_or_sync(FULLMASK, died_nocap);
        D.bad |= __reduce_or_sync(FULLMASK, died_bad);
    }
    if (x.prof_on) x.t_epi += clock64() - tq2;
    __syncwarp();
}

// ---- k_pack: node-sorted claims (output of the bucketing kernels), one warp per node -------------------
// dynamic smem per CTA: [tbl 1024][tbar 16][per warp: inv 512 | ring 2048 | live 1024+128 | bars 48]
constexpr uint32_t PK_TBL = 0, PK_TBAR = 1024, PK_WARP0 = 1040, PK_INV = 0, PK_RING = 512, PK_LIVE = 2560,
                   PK_BARS = 3712, PK_WSTRIDE = 3760;      // live = 1024 B records + 128 B results
__host__ __device__ constexpr uint32_t pack_smem_bytes(int wpc) { return PK_WARP0 + (uint32_t)wpc * PK_WSTRIDE; }

// claim m of the node's span from the shared-memory ring (all lanes read one address: broadcast)
struct RingGet {
    uint32_t ring_addr; uint32_t segbase;
    __device__ __forceinline__ uint4 operator()(uint32_t m) const {
        return lds128(ring_addr + ((((segbase + (m >> 5)) & (RING - 1)) * SEG + (m & 31)) << 4));
    }
};

// Every load that does not depend on another is issued before the first wait: the bench flushes L2, so each
// dependent round trip is a DRAM (or at best L2) latency.
template <int WPC>
__global__ void __launch_bounds__(WPC * 32, 1)
k_pack(const PackArgs a) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const uint32_t sbase = smem_base(dyn_smem);
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t wbase = sbase + PK_WARP0 + wid * PK_WSTRIDE;
    const uint32_t ring_addr = wbase + PK_RING, bar_addr = wbase + PK_BARS, inv_addr = wbase + PK_INV;
    const uint32_t tbar_addr = sbase + PK_TBAR;

    if (lane == 0) {
        #pragma unroll
        for (int q = 0; q <= (int)RING; ++q) mbar_init_a(bar_addr + q * 8, 1);
        if (wid == 0) mbar_init_a(tbar_addr, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) tma_load_a(sbase + PK_TBL, a.tbl, 1024u, tbar_addr);   // placement table, waited on later
    pdl_wait();                                    // sorted claims / claim_off come from the bucketing kernels
    bool tbl_ready = false;

    NodeCtx x;
    x.lane = lane; x.ltmask = lanemask_lt();
    x.live_addr = wbase + PK_LIVE; x.tbl_addr = sbase + PK_TBL;
    x.tbl_ptr = reinterpret_cast<const uint32_t*>(dyn_smem + PK_TBL);
    x.have_off = a.have_off != 0;
    x.sc = a.sel;
    x.sink = OutSink{a.out, a.n_out, a.err, lane};

    uint32_t segbase = 0;      // running segment counter: ring slot = (segbase+q) % RING
    uint32_t inv_phase = 0;
    const uint32_t nwarps = gridDim.x * WPC;
    for (uint32_t node = blockIdx.x * WPC + wid; node < a.n_node; node += nwarps) {
        // one round trip: the node's extents and the upstream error flag
        const uint32_t g0 = __ldg(&a.node_off[node]);
        const uint32_t g1 = __ldg(&a.node_off[node + 1]);
        const uint32_t c0 = __ldg(&a.claim_off[node]);
        const uint32_t c1 = __ldg(&a.claim_off[node + 1]);
        const uint32_t bad_input = a.err.dev[ERR_NOT_SORTED];
        const uint32_t ng = g1 - g0, cnt = c1 - c0;
        if (bad_input) return;                  // input contract violated upstream: leave the inventory alone
        if (cnt == 0) {
            if (a.inv_src != a.inv_dst && lane < ng) a.inv_dst[g0 + lane] = __ldg(&a.inv_src[g0 + lane]);
            continue;
        }
        const uint32_t nseg = (cnt + SEG - 1) / SEG;
        uint32_t issued = 0;
        auto issue = [&](uint32_t q) {
            if (lane == 0) {
                const uint32_t slot = (segbase + q) & (RING - 1);
                tma_load_a(ring_addr + slot * SEG * 16, a.sorted + c0 + q * SEG, min(SEG, cnt - q * SEG) * 16u, bar_addr + slot * 8);
            }
        };
        // second round trip: GpuRecs + first claim segments, all in flight at once
        if (lane == 0 && ng) tma_load_a(inv_addr, a.inv_src + g0, ng * 16u, bar_addr + RING * 8);
        while (issued < nseg && issued < 3) issue(issued++);
        if (!tbl_ready) { mbar_wait_a(tbar_addr, 0); tbl_ready = true; }

        uint4 rec = make_uint4(0, 0, 0, 0);
        if (ng) { mbar_wait_a(bar_addr + RING * 8, inv_phase); inv_phase ^= 1; if (lane < ng) rec = lds128(inv_addr + lane * 16); }
        x.g0 = g0;
        x.begin(rec, lane < ng);
        RingGet get{ring_addr, segbase};

        uint32_t waited = 0;
        for (uint32_t seg = 0; seg < nseg; ++seg) {
            const uint32_t need = min(nseg - 1, seg + 1);           // current + look-ahead for runs
            while (waited <= need) {
                mbar_wait_a(bar_addr + ((segbase + waited) & (RING - 1)) * 8, ((segbase + waited) / RING) & 1);
                ++waited;
            }
            __syncwarp();
            while (issued < nseg && issued <= seg + 2) issue(issued++);   // slot of seg-1 is free by now
            const uint32_t n_in = min(SEG, cnt - seg * SEG);
            const uint32_t slot = (segbase + seg) & (RING - 1);
            uint4 c = make_uint4(0xFFu, 0, 0, 0);
            if (lane < n_in) c = lds128(ring_addr + ((slot * SEG + lane) << 4));
            segment_run(x, c, lane < n_in, seg * SEG + lane, get, cnt);
        }
        if (lane < ng) a.inv_dst[g0 + lane] = x.L.store(rec);
        segbase += nseg;
        __syncwarp();
    }
}

// ---- k_fused: the whole Allocate batch in ONE launch, for batches where n_node * n_claim is small --------
// One CTA of NW warps per node.  All warps stream the claim array (each its own contiguous part, so every
// warp's matches are in input order) and keep the indices of the claims that select this node; then warp 0
// packs them.  No sort, no sorted copy, no claim_off: the O(n_node * n_claim) key tests are spread over
// n_node SMs and every byte after the first CTA's touch comes from L2.
// dynamic smem: [tbl 1024][bars 16][inv 512][live 1024+128][counts 64][index lists: n_claim u32, warp w at w*chunk]
constexpr uint32_t FU_TBL = 0, FU_TBAR = 1024, FU_IBAR = 1032, FU_INV = 1040, FU_LIVE = 1552, FU_CNT = 2704, FU_LIST = 2832;   // counts: up to 32 warps
constexpr uint32_t FU_PIECE = 256;          // claims per staged piece: one warp's 8 loads of 32 claims
constexpr uint32_t FU_MAXPIECE = 8;         // pieces per warp part => staging needs n_claim <= NW * 2048
// per-warp part of the claim array: a multiple of 32 claims, of a whole piece when the array is staged
__host__ __device__ constexpr uint32_t fused_chunk(uint32_t n_claim, int nw, bool stage) {
    return stage ? ((n_claim + nw * FU_PIECE - 1) / (nw * FU_PIECE)) * FU_PIECE
                 : ((n_claim + nw * 32 - 1) / (nw * 32)) * 32;
}
__host__ __device__ constexpr size_t fused_list_bytes(uint32_t n_claim, int nw, bool stage) {
    return (size_t)fused_chunk(n_claim, nw, stage) * nw * 4;
}
// (staged: the NW * FU_MAXPIECE * 8 bytes in front of the index lists are unused, kept so the staged capacity stays 11,117 claims)
__host__ __device__ constexpr size_t fused_smem_bytes(uint32_t n_claim, int nw, bool stage) {
    return FU_LIST + (stage ? (size_t)nw * FU_MAXPIECE * 8 : 0) + fused_list_bytes(n_claim, nw, stage) + 16 + (stage ? (size_t)n_claim * 16 + 16 : 0);
}

template <int NW>
struct IdxGet {            // claim m of the node, through the index lists
    const uint4* claims; const uint32_t* out_off; uint32_t list_addr, chunk; uint32_t pre[NW];
    uint32_t stage_addr;   // != 0: the whole claim array is staged in shared memory at this address
    __device__ __forceinline__ uint32_t index_of(uint32_t m) const {
        uint32_t w = 0;
        #pragma unroll
        for (int i = 1; i < NW; ++i) w += m >= pre[i];
        uint32_t base = 0;
        #pragma unroll
        for (int i = 1; i < NW; ++i) base = (w == (uint32_t)i) ? pre[i] : base;
        return lds32(list_addr + ((w * chunk + (m - base)) << 2));
    }
    __device__ __forceinline__ uint4 operator()(uint32_t m) const {
        const uint32_t i = index_of(m);
        uint4 c = stage_addr ? lds128(stage_addr + (i << 4)) : __ldg(&claims[i]);
        c.y = out_off ? __ldcg(&out_off[i]) : i;
        return c;
    }
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
#define DRA_DSTAMP(k) do { if (a.timeline && blockIdx.x == 0 && threadIdx.x == 0) a.timeline[(a.n_node + 2) * 8 + (k)] = globaltimer_ns(); } while (0)
#define DRA_TSTAMP(k) do { if (a.timeline && threadIdx.x == 0) a.timeline[(a.n_node + 4) * 8 + blockIdx.x * 8 + (k)] = globaltimer_ns(); } while (0)
#define DRA_STAMP(k) do { if (a.timeline && threadIdx.x == 0) a.timeline[blockIdx.x * 8 + (k)] = (k) == 0 ? globaltimer_ns() : (unsigned long long)clock64(); } while (0)

// Grid-wide barrier for a cooperative launch (all CTAs resident).  Sense-free: the last arriver resets the count
// and bumps the generation the others spin on, so the two words are reusable across barriers and launches.
// bar.sync orders the CTA's earlier stores before thread 0's fence (fences are cumulative); a bounded spin turns a
// lost CTA into an error flag instead of a hang.
__device__ __forceinline__ void grid_barrier(uint32_t* gbar, uint32_t n_cta, const Err& err) {
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t gen;
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(gen) : "l"(gbar + 1) : "memory");
        __threadfence();
        if (atomicAdd(gbar, 1u) == n_cta - 1) {
            gbar[0] = 0;
            __threadfence();
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(gbar + 1), "r"(gen + 1) : "memory");
        } else {
            const long long t0 = clock64();
            uint32_t v;
            do {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(gbar + 1) : "memory");
                if (v != gen) break;
                if (clock64() - t0 > 400000000ll) { err.set(ERR_DEVICE_WAIT); break; }
            } while (true);
        }
    }
    __syncthreads();
}

// The body of the single-launch kernel: one batch.  k_fused runs it once; k_serve (resident mode) runs it once per doorbell
// (`again`: the shared-memory barriers of the previous batch are invalidated first).
// What differs from batch to batch (resident mode keeps everything else in the kernel's parameter space)
struct Batch {
    uint32_t n_claim, n_out, have_off;
    const uint4* inv_src;
    const uint32_t* out_off;
    const uint4* h_claims; const uint32_t* h_out_off; uint2* h_out;
};

template <int NW, bool STAGE>
__device__ __forceinline__ void fused_body(const PackArgs& a, const Batch b, uint8_t* dyn_smem, const bool again) {
    DRA_STAMP(0); DRA_STAMP(1); DRA_TSTAMP(0);
    const uint32_t sbase = smem_base(dyn_smem);
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t node = blockIdx.x;
    const bool has_node = node < a.n_node;       // CTA n_node handles claims that name no node
    const uint32_t tbar = sbase + FU_TBAR, ibar = sbase + FU_IBAR;
    const uint32_t list_addr = sbase + FU_LIST + (STAGE ? (uint32_t)NW * FU_MAXPIECE * 8u : 0u);
    const uint32_t stage_addr = STAGE ? ((list_addr + (uint32_t)fused_list_bytes(b.n_claim, NW, STAGE) + 15u) & ~15u) : 0u;
    // multi-GPU send queue: behind everything else of the layout; [q_cap entries of 16 B]; its counter and end marker
    // live in the spare words of the counts area
    const uint32_t q_base = (sbase + (uint32_t)fused_smem_bytes(b.n_claim, NW, STAGE) + 15u) & ~15u;
    const uint32_t q_cnt_addr = sbase + FU_CNT + 104, q_done_addr = sbase + FU_CNT + 108;
    const bool q_on = a.peer.world != 0 && a.q_cap != 0 && has_node;
    const uint32_t q_tag = a.peer.epoch | 0x80000000u;
    if (q_on) {                                   // clear the tags (shared memory holds garbage at launch)
        for (uint32_t e = threadIdx.x; e < a.q_cap; e += NW * 32) sts128(q_base + (e << 4), make_uint4(0, 0, 0, 0));
        if (threadIdx.x == 0) { sts32(q_cnt_addr, 0); sts32(q_done_addr, 0xFFFFFFFFu); }
    }
    // round trip 1: extents (needed for the inventory copy); table copy goes out immediately
    uint32_t g0 = 0, g1 = 0;
    if (has_node) { g0 = __ldg(&a.node_off[node]); g1 = __ldg(&a.node_off[node + 1]); }
    // the table and inventory barriers, then one fence + sync
    if (again) {                                   // resident mode: the previous batch's barriers are dead objects now
        // warp 0 wrote this node's GpuRecs with generic stores in the previous batch; the bulk copy below reads them
        // through the async proxy
        asm volatile("fence.proxy.async;" ::: "memory");
        __syncthreads();
        if (threadIdx.x == 0) { mbar_inval_a(tbar); mbar_inval_a(ibar); }
        __syncthreads();
    }
    if (threadIdx.x == 0) { mbar_init_a(tbar, 1); mbar_init_a(ibar, 1); }
    mbar_fence_init();
    __syncthreads();
    if (threadIdx.x == 0) tma_load_a(sbase + FU_TBL, a.tbl, 1024u, tbar);
    const uint32_t ng = g1 - g0;
    if (threadIdx.x == 32 && ng) tma_load_a(sbase + FU_INV, b.inv_src + g0, ng * 16u, ibar);
    // sharded call: the claim list was compacted on the device by the kernel before this one; b.n_claim is its capacity
    if (a.sh_on) {
        // ... or right here: one 1024-claim tile per CTA (cooperative launch), a grid barrier, and the list is there —
        // no second launch; the table and inventory copies above are already in flight behind it
        if (blockIdx.x < a.sh.n_tiles) shard_tile_flat<SC_IN_ROWS>(a.sh, blockIdx.x);
        grid_barrier(a.dio.gbar, gridDim.x, a.err);
    }
    else if (a.n_dev) pdl_wait();                            // (launched as a programmatic dependent of the compaction)
    const uint32_t n_claim = a.n_dev ? min(b.n_claim, __ldcg(a.n_dev)) : b.n_claim;
    if (a.n_dev && __ldcg(a.n_dev) > b.n_claim) {            // laid out for fewer claims: touch nothing, tell everybody
        if (blockIdx.x == 0) {
            if (threadIdx.x == 0) a.err.set(ERR_SHARD_PLAN);
            if (a.peer.world) { pkt_send_header(a.peer, threadIdx.x, 0xFFFFFFFFu); if (threadIdx.x == 32) a.peer.cursor[a.peer.parity ^ 1u] = 0; }
        }
        return;
    }

    if (STAGE && b.h_claims) {
        // direct ingest: one 16-byte load from the caller's pinned buffer per thread (a single PCIe round trip for
        // the whole grid), stored to the device copy that every CTA's filter below reads from L2.
        // (Per-piece ready flags instead of the grid barrier were tried while the stage was filled by bulk copies: slower
        // — every producer then pays its own fence on the critical path.)
        DRA_DSTAMP(0);
        const uint32_t nthr = gridDim.x * (NW * 32), t0 = blockIdx.x * (NW * 32) + threadIdx.x;
        for (uint32_t i = t0; i < b.n_claim; i += nthr) a.dio.d_claims[i] = __ldcs(b.h_claims + i);
        if (b.h_out_off) for (uint32_t i = t0; i < b.n_claim; i += nthr) a.dio.d_out_off[i] = __ldcs(b.h_out_off + i);
        DRA_DSTAMP(1);
        grid_barrier(a.dio.gbar, gridDim.x, a.err);
        DRA_DSTAMP(2);
    }
    DRA_STAMP(2);

    const uint32_t chunk = fused_chunk(n_claim, NW, STAGE);            // per-warp part of the filter
    const uint32_t lo = wid * chunk, hi = min(n_claim, lo + chunk);
    // STAGE: each lane loads whole claims into registers, tests the key there and stores the claim into the stage, from
    // which the pack, the stray CTA and the tail read it after the filter's __syncthreads.  (Filling the stage with
    // 4 KiB bulk copies instead left the filter waiting for them to be issued and land: profiles/timeline.py.)
    // L2-coherent loads only: the array may have been written inside this launch by other CTAs (direct-I/O ingest,
    // in-kernel compaction) or, in k_serve, rewritten for this batch while the kernel stayed up.
    // The first 8 claims of every lane go out now, so warp 0's are in flight while it waits for the table and GpuRecs.
    constexpr int U = 8;
    const uint4 none = make_uint4(0u, 0xFFFFFFFFu, 0u, 0u);
    uint4 cur[U];
    if (STAGE) {
        #pragma unroll
        for (int u = 0; u < U; ++u) { const uint32_t i = lo + u * 32 + lane; cur[u] = i < hi ? __ldcg(a.claims + i) : none; }
    }

    // warp 0 sets up the node (inventory, table row properties) NOW: it needs only the table and the GpuRecs, in flight
    // since the entry — after the filter this would sit on the critical path
    NodeCtx x;
    uint4 rec = make_uint4(0, 0, 0, 0);
    if (wid == 0 && has_node) {
        x.lane = lane; x.ltmask = lanemask_lt();
        x.live_addr = sbase + FU_LIVE; x.tbl_addr = sbase + FU_TBL;
        x.tbl_ptr = reinterpret_cast<const uint32_t*>(dyn_smem + FU_TBL);
        x.have_off = b.have_off != 0;
        x.sc = a.sel;
        x.sink = OutSink{a.out, b.n_out, a.err, lane};
        x.g0 = g0;
        mbar_wait_a(tbar, 0);
        if (ng) { mbar_wait_a(ibar, 0); if (lane < ng) rec = lds128(sbase + FU_INV + lane * 16); }
        x.begin(rec, lane < ng);
    }

    // ---- filter: which claims select this node (all warps) ------------------------------------------
    const uint32_t ltmask = lanemask_lt();
    const uint32_t my_list = list_addr + (lo << 2);
    const uint32_t want = has_node ? node : 0xFFFFFFFEu;
    const bool stray_cta = node == a.n_node;
    uint32_t cntw = 0, slot_l = 0;                                     // slot_l: OutRec slots of this lane's matches (gather only)
    const bool gather = a.peer.world != 0;
    // one claim per lane; warp-uniform control flow.  xv: the claim's first word (STAGE only, loaded with the key)
    auto scan = [&](const uint32_t i, const uint32_t keyv, const uint32_t xv) {
        // CTA n_node collects the claims that name no node of the inventory (they become INVALID, spec §3)
        const bool m = has_node ? keyv == want : (stray_cta && i < hi && keyv >= a.n_node);
        const uint32_t bm = __ballot_sync(FULLMASK, m);
        if (bm) {
            if (m) {
                sts32(my_list + ((cntw + (uint32_t)__popc(bm & ltmask)) << 2), i);
                if (gather) {                                          // the packet range is reserved while the pack runs
                    const uint32_t x_ = STAGE ? xv : __ldg(reinterpret_cast<const uint32_t*>(a.claims) + 4 * (size_t)i);
                    const uint32_t kind = x_ & 0xFFu, count = x_ >> 16;
                    slot_l += (!stray_cta && kind == DRA_KIND_GPU && !claim_invalid(kind, 0, count, b.have_off != 0)) ? count : 1u;
                }
            }
            cntw += (uint32_t)__popc(bm);
        }
    };
    if (STAGE) {                                                       // (the first 8 claims were issued above)
        uint4 nxt[U];
        for (uint32_t base = lo; base < hi; base += 32 * U) {
            #pragma unroll
            for (int u = 0; u < U; ++u) {                      // next batch goes out before this one is looked at
                const uint32_t i = base + 32 * U + u * 32 + lane;
                nxt[u] = i < hi ? __ldcg(a.claims + i) : none;
            }
            #pragma unroll
            for (int u = 0; u < U; ++u) {
                const uint32_t i = base + u * 32 + lane;
                if (i < hi) sts128(stage_addr + (i << 4), cur[u]);
                scan(i, cur[u].y, cur[u].x);
            }
            #pragma unroll
            for (int u = 0; u < U; ++u) cur[u] = nxt[u];
        }
    } else {
        const uint32_t* keyp = reinterpret_cast<const uint32_t*>(a.claims) + 1;      // .y of claim i at keyp[4*i]
        uint32_t key[U], nxt[U];
        #pragma unroll
        for (int u = 0; u < U; ++u) { const uint32_t i = lo + u * 32 + lane; key[u] = i < hi ? __ldg(keyp + 4 * (size_t)i) : 0xFFFFFFFFu; }
        for (uint32_t base = lo; base < hi; base += 32 * U) {
            #pragma unroll
            for (int u = 0; u < U; ++u) {                      // next batch goes out before this one is looked at
                const uint32_t i = base + 32 * U + u * 32 + lane;
                nxt[u] = i < hi ? __ldg(keyp + 4 * (size_t)i) : 0xFFFFFFFFu;
            }
            #pragma unroll
            for (int u = 0; u < U; ++u) scan(base + u * 32 + lane, key[u], 0u);
            #pragma unroll
            for (int u = 0; u < U; ++u) key[u] = nxt[u];
        }
    }
    DRA_STAMP(3);
    if (lane == 0) sts32(sbase + FU_CNT + (wid << 2), cntw);
    if (gather) { slot_l = __reduce_add_sync(FULLMASK, slot_l); if (lane == 0) sts32(sbase + FU_CNT + 64 + (wid << 2), slot_l); }
    __syncthreads();
    if (gather && threadIdx.x == NW * 32 - 1) {    // one reservation per CTA, issued now: its round trip hides behind the pack
        uint32_t tot = 0;
        #pragma unroll
        for (int i = 0; i < NW; ++i) tot += lds32(sbase + FU_CNT + 64 + (i << 2));
        sts32(sbase + FU_CNT + 100, tot);
        sts32(sbase + FU_CNT + 96, tot ? atomicAdd(&a.peer.cursor[a.peer.parity], tot) : 0u);
    }
    // every record of this node fits the send queue: the idle warps send while warp 0 packs
    bool use_q = false;
    if (q_on) {
        uint32_t tot = 0;
        #pragma unroll
        for (int i = 0; i < NW; ++i) tot += lds32(sbase + FU_CNT + 64 + (i << 2));
        use_q = tot != 0 && tot <= a.q_cap;
    }
    DRA_STAMP(4);

    IdxGet<NW> get;
    get.claims = a.claims; get.out_off = b.out_off; get.list_addr = list_addr; get.chunk = chunk;
    get.stage_addr = stage_addr;
    uint32_t cnt = 0;
    #pragma unroll
    for (int i = 0; i < NW; ++i) { get.pre[i] = cnt; cnt += lds32(sbase + FU_CNT + (i << 2)); }

    if (stray_cta) {                               // claims naming no node: INVALID (spec §3); no state is touched
        for (uint32_t m = threadIdx.x; m < cnt; m += NW * 32) {
            const uint32_t i = get.index_of(m);
            const uint4 c = STAGE ? lds128(stage_addr + (i << 4)) : __ldcg(&a.claims[i]);
            const uint32_t dst = b.out_off ? __ldcg(&b.out_off[i]) : i;
            const uint32_t kind = c.x & 0xFFu;
            const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : ((c.x >> 8) & 0xFFu);
            if (dst < b.n_out) a.out[dst] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, DRA_ST_INVALID));
            else a.err.set(ERR_OUT_RANGE);
        }
    }
    // ---- pack: warp 0 ----------------------------------------------------------------------------------
    if (wid == 0 && has_node) {
        if (cnt == 0) {
            if (b.inv_src != a.inv_dst && lane < ng) a.inv_dst[g0 + lane] = __ldg(&b.inv_src[g0 + lane]);
        } else {
            // the first segment's claims are requested before waiting for the table / inventory
            auto fetch = [&](uint32_t seg, uint4& c, bool& present) {
                const uint32_t m = seg * SEG + lane;
                present = m < cnt;
                c = make_uint4(0xFFu, 0, 0, 0);
                if (present) c = get(m);
            };
            uint4 c_cur; bool p_cur;
            fetch(0, c_cur, p_cur);

            x.prof_on = a.timeline != nullptr;
            if (use_q) { x.sink.q_addr = q_base; x.sink.q_cap = a.q_cap; x.sink.q_cnt = q_cnt_addr; x.sink.q_tag = q_tag; }
            DRA_STAMP(5);

            const uint32_t nseg = (cnt + SEG - 1) / SEG;
            for (uint32_t seg = 0; seg < nseg; ++seg) {
                uint4 c_nxt = make_uint4(0xFFu, 0, 0, 0); bool p_nxt = false;
                const long long tf0 = x.prof_on ? clock64() : 0;
                if (seg + 1 < nseg) fetch(seg + 1, c_nxt, p_nxt);       // in flight while this segment is packed
                if (x.prof_on) x.t_fetch += clock64() - tf0;
                segment_run(x, c_cur, p_cur, seg * SEG + lane, get, cnt);
                c_cur = c_nxt; p_cur = p_nxt;
            }
            if (lane < ng) a.inv_dst[g0 + lane] = x.L.store(rec);
            if (use_q) {                               // the senders may leave after this many
                __syncwarp();
                if (lane == 0) { const uint32_t put_ = lds32(q_cnt_addr); sts32(q_done_addr, put_); if (put_ > a.q_cap) a.err.set(ERR_PEER_TIMEOUT); }
            }
            DRA_STAMP(6);
            if (a.timeline && lane == 0) {
                a.timeline[blockIdx.x * 8 + 7] = (cnt & 0xFFFFu) | ((unsigned long long)(x.n_live & 0xFFFFu) << 16) |
                    ((unsigned long long)(x.t_fetch & 0xFFFF) << 32) | ((unsigned long long)(x.t_pre_a & 0xFFFF) << 48);
                a.timeline[blockIdx.x * 8 + 0] = (unsigned long long)x.t_pre | ((unsigned long long)x.t_loop << 20) | ((unsigned long long)x.t_epi << 40);
            }
        }
    }
    if (use_q && wid != 0) {
        // the senders: warps 1..NW-1.  Entry e of the queue becomes packet (base + e) of this rank's slice at every peer.
        asm volatile("bar.sync 1, %0;" ::"n"((NW - 1) * 32) : "memory");     // the reservation (last thread) is visible
        const uint32_t base = lds32(sbase + FU_CNT + 96);
        const PktGather& pg = a.peer;
        for (uint32_t e = threadIdx.x - 32; ; e += (NW - 1) * 32) {
            uint4 v; bool have = false;
            while (true) {
                if (e < a.q_cap) { v = lds128(q_base + (e << 4)); if (v.w == q_tag) { have = true; break; } }
                const uint32_t dn = lds32(q_done_addr);
                if (dn != 0xFFFFFFFFu && e >= dn) break;
                __nanosleep(40);
            }
            if (!have) break;
            if (base + e < pg.cap) pkt_send(pg, base + e, make_uint2(v.x, v.y), pg.slot_base + v.z);
        }
    }
    if (STAGE && b.h_claims) {
        // direct egress: when every CTA's OutRecs are in the device buffer, the grid writes them to the caller's
        // pinned buffer as coalesced 16-byte stores (a scattered 8-byte store per record is what makes plain
        // zero-copy output slow: profiles/e2e_parts.py)
        DRA_DSTAMP(3);
        grid_barrier(a.dio.gbar, gridDim.x, a.err);
        DRA_DSTAMP(4);
        const uint32_t nthr = gridDim.x * (NW * 32), t0 = blockIdx.x * (NW * 32) + threadIdx.x;
        const uint32_t n16 = b.n_out >> 1;
        const uint4* src = reinterpret_cast<const uint4*>(a.out);
        uint4* dst = reinterpret_cast<uint4*>(b.h_out);
        for (uint32_t i = t0; i < n16; i += nthr) __stcs(dst + i, __ldcg(src + i));
        if ((b.n_out & 1u) && t0 == 0) b.h_out[b.n_out - 1] = __ldcg(a.out + b.n_out - 1);
        DRA_DSTAMP(5);
        return;
    }
    if (a.peer.world == 0) return;

    // ---- multi-GPU tail: the all-gather, fused here (no extra launch, no fence, no flag) -----------------------
    // 1. every CTA sends the OutRecs of ITS node's claims as packets into a contiguous range of this rank's slice at
    //    every peer; 2. every CTA then polls its share of the peers' slices in local memory and fills the table.
    __syncthreads();                                   // warp 0's OutRecs are visible to the whole CTA
    DRA_TSTAMP(1);
    const PktGather& pg = a.peer;
    __shared__ uint32_t pk_next_s;
    if (threadIdx.x == 0) pk_next_s = 0;
    if (blockIdx.x == 0 && threadIdx.x == 32) pg.cursor[pg.parity ^ 1u] = 0;       // the next call's cursor
    __syncthreads();
    // the claims this CTA answers for: its node's list, or (CTA n_node) the claims that name no node (one slot each)
    auto slots_of = [&](const uint4 c) -> uint32_t {
        const uint32_t kind = c.x & 0xFFu, count = c.x >> 16;
        return (!stray_cta && kind == DRA_KIND_GPU && !claim_invalid(kind, 0, count, b.have_off != 0)) ? count : 1u;
    };
    auto claim_at = [&](uint32_t i) -> uint4 { return STAGE ? lds128(stage_addr + (i << 4)) : __ldcg(&a.claims[i]); };
    // (the range [base, base + total) of this rank's slice was reserved right after the filter)
    const uint32_t pk_total = lds32(sbase + FU_CNT + 100), pk_base = lds32(sbase + FU_CNT + 96);
    if (pk_total && !use_q) {
        const uint32_t base = pk_base;
        for (uint32_t m = threadIdx.x; m < cnt; m += NW * 32) {
            const uint32_t i = get.index_of(m);
            const uint32_t dst = b.out_off ? __ldcg(&b.out_off[i]) : i, sl = slots_of(claim_at(i));
            if (dst > b.n_out || sl > b.n_out - dst) continue;
            const uint32_t at = base + atomicAdd(&pk_next_s, sl);
            for (uint32_t s_ = 0; s_ < sl; ++s_)
                if (at + s_ < pg.cap) pkt_send(pg, at + s_, __ldcg(a.out + dst + s_), pg.slot_base + dst + s_);
        }
    }
    DRA_TSTAMP(2);
    pkt_finish_send(pg);                               // the last CTA to get here tells the peers how many packets went out
    DRA_TSTAMP(3);
    pkt_receive(pg, blockIdx.x * (NW * 32) + threadIdx.x, gridDim.x * (NW * 32), a.err);
    __syncthreads();
    DRA_TSTAMP(4);
}

template <int NW, bool STAGE>
__global__ void __launch_bounds__(NW * 32, 1)
k_fused(const PackArgs a) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    const Batch b{a.n_claim, a.n_out, a.have_off, a.inv_src, a.out_off, a.dio.h_claims, a.dio.h_out_off, a.dio.h_out};
    fused_body<NW, STAGE>(a, b, dyn_smem, false);
}

// ---- resident mode: the kernel stays up and takes batches by DOORBELL ------------------------------------------------
// Much of a host call through a cooperative launch is the launch and the stream synchronisation.  Here the kernel is launched once; a call is: the host writes a 64-byte command (sizes, flags, the pinned buffers) into
// mapped host memory, then its sequence number; CTA 0 polls that word, relays the command through L2, every CTA runs
// the batch body with direct host I/O (ingest -> barrier -> filter + pack -> barrier -> egress), and after a system fence
// per CTA and a last grid barrier CTA 0 writes the sequence number into the host's completion word.  No launch, no
// stream call, no driver call on the host at all.  The kernel leaves on an EXIT command or after `idle` cycles without
// a doorbell (the host relaunches on demand), so it can never outlive its owner by more than that.
struct ServeCmd {                 // one cache line of mapped host memory, written by the host
    uint32_t seq, n_claim, n_out, flags;         // flags: DRA_F_FRESH_INVENTORY | SERVE_EXIT
    unsigned long long claims, out_off, out;     // pinned host buffers of this batch (device-visible addresses)
    unsigned long long pad[3];
};
constexpr uint32_t SERVE_EXIT = 0x80000000u;
struct ServeArgs {
    PackArgs base;                // inventory, table, node_off, err, selectors, device copies (dio.d_claims ...), dio.gbar
    const uint4* inv_pristine;
    const volatile ServeCmd* h_cmd;              // device view of the command line
    volatile uint32_t* h_stat;                   // [0] completed seq, [1] state: 1 running, 2 exited, [2] exit reason
    uint32_t* d_go;                              // device: [0] sequence relayed by CTA 0, [4..19] the command copy
    uint32_t first_seq, cap_claims;
    long long idle_cycles;
};

template <int NW>
__global__ void __launch_bounds__(NW * 32, 1)
k_serve(const ServeArgs s) {
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    __shared__ uint32_t cmd_s[12];
    uint32_t seq = s.first_seq;
    bool again = false;
    if (blockIdx.x == 0 && threadIdx.x == 0) { s.h_stat[1] = 1u; __threadfence_system(); }
    for (;;) {
        if (blockIdx.x == 0 && threadIdx.x < 32) {
            // the doorbell: lanes 0..3 read 16 bytes each of the 64-byte command line — ONE PCIe read per poll brings the
            // sequence number AND the whole command (the host writes the fields first, the sequence number last)
            const long long t0 = clock64();
            uint4 h = make_uint4(0, 0, 0, 0); bool quit = false;
            for (;;) {
                if (threadIdx.x < 4)
                    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(h.x), "=r"(h.y), "=r"(h.z), "=r"(h.w)
                                 : "l"((const uint4*)(const void*)const_cast<const ServeCmd*>(s.h_cmd) + threadIdx.x) : "memory");
                const uint32_t got = __shfl_sync(FULLMASK, h.x, 0);
                if (got == seq) break;
                if (clock64() - t0 > s.idle_cycles) { quit = true; break; }
            }
            if (threadIdx.x == 0 && !quit && !(h.w & SERVE_EXIT)) reinterpret_cast<unsigned long long*>(s.d_go + 32)[0] = globaltimer_ns();    // instrumentation: doorbell seen
            uint32_t* c = s.d_go + 4;
            if (threadIdx.x < 4) {
                if (quit) { if (threadIdx.x == 0) { c[0] = seq; c[1] = 0; c[2] = 0; c[3] = SERVE_EXIT | 1u; } }
                else *reinterpret_cast<uint4*>(c + 4 * threadIdx.x) = h;      // {seq,n,n_out,flags} {claims,out_off} {out,-}
            }
            __syncwarp();
            if (threadIdx.x == 0) { __threadfence(); asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(s.d_go), "r"(seq) : "memory"); }
        }
        if (threadIdx.x == 0) {
            uint32_t v;
            do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(s.d_go) : "memory"); } while (v != seq);
            #pragma unroll
            for (int k = 0; k < 10; ++k) cmd_s[k] = __ldcg(s.d_go + 4 + k);
        }
        __syncthreads();
        const uint32_t n_claim = cmd_s[1], n_out = cmd_s[2], flags = cmd_s[3];
        if (flags & SERVE_EXIT) {
            if (blockIdx.x == 0 && threadIdx.x == 0) { s.h_stat[2] = flags & 1u; s.h_stat[1] = 2u; __threadfence_system(); }
            return;
        }
        const PackArgs& a = s.base;
        Batch b;
        b.n_claim = n_claim; b.n_out = n_out;
        b.inv_src = (flags & DRA_F_FRESH_INVENTORY) ? s.inv_pristine : const_cast<const uint4*>(s.base.inv_dst);
        b.h_claims = reinterpret_cast<const uint4*>(((unsigned long long)cmd_s[5] << 32) | cmd_s[4]);
        b.h_out_off = reinterpret_cast<const uint32_t*>(((unsigned long long)cmd_s[7] << 32) | cmd_s[6]);
        b.h_out = reinterpret_cast<uint2*>(((unsigned long long)cmd_s[9] << 32) | cmd_s[8]);
        b.out_off = b.h_out_off ? a.dio.d_out_off : nullptr;
        b.have_off = b.h_out_off != nullptr;
        if (n_claim <= s.cap_claims) fused_body<NW, true>(a, b, dyn_smem, again);
        else if (blockIdx.x == 0 && threadIdx.x == 0) a.err.set(ERR_SHARD_PLAN);          // (the host never sends such a batch)
        // completion: every CTA fences its stores to the host's buffers and takes a ticket; the last one tells the host
        // (one word).  Nobody waits here: the next doorbell cannot ring before the host has seen this word.
        __syncthreads();
        if (threadIdx.x == 0) {
            if (blockIdx.x == 0) reinterpret_cast<unsigned long long*>(s.d_go + 32)[1] = globaltimer_ns();        // CTA 0's egress stores issued
            __threadfence_system();
            if (atomicAdd(s.d_go + 2, 1u) == gridDim.x - 1) {
                s.d_go[2] = 0;
                __threadfence();
                reinterpret_cast<unsigned long long*>(s.d_go + 32)[2] = globaltimer_ns();                           // every CTA fenced
                asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(s.h_stat), "r"(seq) : "memory");
                __threadfence_system();
                reinterpret_cast<unsigned long long*>(s.d_go + 32)[3] = globaltimer_ns();                           // completion word out
            }
        }
        ++seq; again = true;
    }
}

// ====================================================================================================
// pod mode (spec §12): atomic evaluation of a pod on one node, with the exhaustive placement search
// ====================================================================================================
// What is searched is the (profile, placement) enumeration deviceLib.getGpuInfo builds per GPU
// (cmd/nvidia-dra-plugin/nvlib.go:244-295, here: the placement table); the multi-request shape is
// demo/specs/quickstart/gpu-test4.yaml:19-44.  The classic driver's recursive search tried one candidate after
// another (SURVEY App. A); here one lane holds one GPU of the node, a level's candidates on ALL GPUs are computed at
// once (shift/AND fit map per lane), a ballot picks the canonical next one (lowest GPU, lowest start), and the
// search stack is two registers per lane: the levels at which this lane's GPU was chosen and the start it got.

// sink of the non-MIG claims of a pod: records go straight to out (rewritten with POD if the pod fails later)
struct PodSink {
    uint2* out; bool failed = false;
    __device__ __forceinline__ bool range(uint32_t, uint32_t) const { return true; }     // checked by k_pod_records
    __device__ __forceinline__ void put(uint32_t idx, uint32_t gpu, uint32_t m) const { if (out) out[idx] = make_uint2(gpu, m); }
    __device__ __forceinline__ bool in_range(uint32_t) const { return true; }
    __device__ __forceinline__ void fail(uint32_t, uint32_t, uint32_t, uint32_t) { failed = true; }
    __device__ __forceinline__ void mark_failed() { failed = true; }
    __device__ __forceinline__ bool stop() const { return failed; }
};

struct PodGet {            // claim m of the pod, .y = its first OutRec slot
    const uint4* pc; const uint32_t* slot; uint32_t base;
    __device__ __forceinline__ uint4 operator()(uint32_t m) const {
        uint4 c = __ldg(&pc[m]);
        c.y = slot ? __ldg(&slot[m]) : base + m;
        return c;
    }
};

// Evaluates the pod pc[0..cnt) (cnt <= 32) on the node whose GPUs sit on the W lanes gbase.. of this warp.
// Returns 0 when the pod was placed (L updated, OutRecs written when out != nullptr), else the failure status
// (L untouched, every slot of the pod rewritten with it / INVALID).  All lanes of the group must call it together.
template <int W>
__device__ __noinline__ uint32_t pod_eval(Lane& L, const uint32_t lane, const uint32_t gmask, const uint32_t gbase,
                                          const uint32_t g0, const uint32_t* __restrict__ tbl_s, const PodGet get,
                                          const uint32_t cnt, const SelCtx sc, const bool exhaustive, const bool have_off,
                                          uint2* __restrict__ out) {
    constexpr uint32_t BLOCKED = DRA_GPU_MIG_ENABLED | DRA_GPU_FULL_ALLOCATED | DRA_GPU_UNAVAILABLE;
    constexpr int R = 32 / W;
    const uint32_t gl = lane - gbase;
    const Lane L0 = L;
    // ---- 1. classify, lane-parallel: lane gl looks at claims gl, gl+W, ... ----
    uint32_t invmask = 0, migmask = 0, grpmask = 0;
    #pragma unroll
    for (int q = 0; q < R; ++q) {
        const uint32_t idx = q * W + gl;
        const bool present = idx < cnt;
        uint4 c = make_uint4(0, 0, 0, 0);
        if (present) c = get(idx);
        const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
        const bool inv = present && (claim_invalid(kind, prof, count, have_off) || claim_sel(kind, c.z, c.w) > sc.n_sel);
        const bool mig = present && kind == DRA_KIND_MIG;
        invmask |= ((__ballot_sync(gmask, inv) & gmask) >> gbase) << (q * W);
        migmask |= ((__ballot_sync(gmask, mig) & gmask) >> gbase) << (q * W);
        grpmask |= ((__ballot_sync(gmask, mig && c.w != 0) & gmask) >> gbase) << (q * W);
    }
    uint32_t status = invmask ? (uint32_t)DRA_ST_POD : 0u;
    // ---- 2. the GPU / SHARED claims, in order, by the default rules (spec §4, §7) ----
    if (!status) {
        PodSink ps{out};
        Dead D;
        uint32_t nm = (cnt >= 32u ? 0xFFFFFFFFu : ((1u << cnt) - 1u)) & ~migmask;
        while (nm && !ps.failed) {
            const uint32_t pos = (uint32_t)__ffs(nm) - 1u; nm &= nm - 1u;
            (void)node_step(L, D, lane, g0, tbl_s, get, pos, cnt, ps, have_off, sc, gmask, gbase);
        }
        if (ps.failed) status = DRA_ST_POD;
    }
    // ---- 3. pre-check: a MIG claim with no placement at all on the node as it stands sinks the pod (one vote per claim) ----
    if (!status) {
        uint32_t mm = migmask;
        while (mm && !status) {
            const uint32_t pos = (uint32_t)__ffs(mm) - 1u; mm &= mm - 1u;
            const uint4 c = get(pos);
            const uint32_t e = tbl_s[L.model * DRA_MAX_PROFILES + ((c.x >> 8) & 0xFFu)];
            bool ok = L.valid && (L.flags & BLOCKED) == DRA_GPU_MIG_ENABLED && (e >> 16) != 0;
            if (c.z != 0) ok = sel_pass(sc, c.z, g0 + gl, L.valid) && ok;
            const bool fits = ok && (fit_map(~L.busy & 0xFFFFu, e & 0xFFu) & (e >> 16)) != 0;
            if (!(__ballot_sync(gmask, fits) & gmask)) status = DRA_ST_POD;
        }
    }
    // ---- the MIG claims: depth-first search in canonical order (GPUs ascending, starts ascending) ----
    uint32_t chosen = 0;                       // bit pos: this lane's GPU holds the claim at position pos
    unsigned long long st_lo = 0, st_hi = 0;   // its start there, one nibble per position
    if (!status && migmask) {
        uint32_t descents = 0, pos = (uint32_t)__ffs(migmask) - 1u;
        uint32_t rl = 0xFFFFFFFFu, rs = 0;     // resume point after a backtrack: candidates after (lane rl, start rs)
        while (true) {
            const uint4 c = get(pos);
            const uint32_t prof = (c.x >> 8) & 0xFFu, group = c.w;
            const uint32_t e = tbl_s[L.model * DRA_MAX_PROFILES + prof];
            const uint32_t smask = e >> 16, size = e & 0xFFu;
            bool ok = L.valid && (L.flags & BLOCKED) == DRA_GPU_MIG_ENABLED && smask != 0;
            if (c.z != 0) ok = sel_pass(sc, c.z, g0 + gl, L.valid) && ok;
            if (group != 0 && (grpmask & ((1u << pos) - 1u))) {                  // co-location: the first earlier member's GPU
                uint32_t be = grpmask & ((1u << pos) - 1u);
                while (be) {
                    const uint32_t j = (uint32_t)__ffs(be) - 1u; be &= be - 1u;
                    if (get(j).w == group) { ok = ok && ((chosen >> j) & 1u); break; }
                }
            }
            uint32_t cand = ok ? (fit_map(~L.busy & 0xFFFFu, size) & smask) : 0u;
            if (rl != 0xFFFFFFFFu) { if (gl < rl) cand = 0; else if (gl == rl) cand &= ~((2u << rs) - 1u); }
            const uint32_t b = __ballot_sync(gmask, cand != 0) & gmask;
            if (b) {
                if (descents == DRA_EXH_BUDGET) { status = DRA_ST_SEARCH_LIMIT; break; }
                ++descents;
                if (lane == (uint32_t)__ffs(b) - 1u) {
                    const uint32_t s_ = (uint32_t)__ffs(cand) - 1u;
                    L.busy |= ((1u << size) - 1u) << s_;
                    chosen |= 1u << pos;
                    if (pos < 16u) st_lo = (st_lo & ~(0xFull << (4u * pos))) | ((unsigned long long)s_ << (4u * pos));
                    else st_hi = (st_hi & ~(0xFull << (4u * (pos - 16u)))) | ((unsigned long long)s_ << (4u * (pos - 16u)));
                }
                const uint32_t rem = pos >= 31u ? 0u : (migmask & ~((2u << pos) - 1u));
                if (!rem) break;                                                  // every level placed
                pos = (uint32_t)__ffs(rem) - 1u; rl = 0xFFFFFFFFu;
            } else {
                const uint32_t below = migmask & ((1u << pos) - 1u);
                if (!exhaustive || !below) { status = DRA_ST_POD; break; }
                pos = 31u - (uint32_t)__clz(below);                               // back to the previous level: undo it
                const uint32_t p2 = (get(pos).x >> 8) & 0xFFu;
                const uint32_t size2 = tbl_s[L.model * DRA_MAX_PROFILES + p2] & 0xFFu;
                const bool mine = (chosen >> pos) & 1u;
                const uint32_t s2 = (uint32_t)((pos < 16u ? st_lo >> (4u * pos) : st_hi >> (4u * (pos - 16u))) & 0xFull);
                const uint32_t wl = __ballot_sync(gmask, mine) & gmask;
                const uint32_t wabs = (uint32_t)__ffs(wl) - 1u;
                if (mine) { L.busy &= ~(((1u << size2) - 1u) << s2); chosen &= ~(1u << pos); }
                rs = __shfl_sync(gmask, s2, wabs);
                rl = wabs - gbase;
            }
        }
    }
    __syncwarp(gmask);
    if (status) {
        L = L0;
        if (out) {                                          // every slot of the pod: INVALID for the malformed claims, else POD / LIMIT
            #pragma unroll
            for (int q = 0; q < R; ++q) {
                const uint32_t idx = q * W + gl;
                if (idx >= cnt) continue;
                const uint4 c = get(idx);
                const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
                const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : prof;
                const uint32_t slots = (kind == DRA_KIND_GPU && !claim_invalid(kind, prof, count, have_off)) ? count : 1u;
                const uint32_t st = ((invmask >> idx) & 1u) ? (uint32_t)DRA_ST_INVALID : status;
                for (uint32_t k = 0; k < slots; ++k) out[c.y + k] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, st));
            }
        }
        return status;
    }
    if (out) {
        uint32_t m = chosen;
        while (m) {
            const uint32_t pos = (uint32_t)__ffs(m) - 1u; m &= m - 1u;
            const uint4 c = get(pos);
            const uint32_t prof = (c.x >> 8) & 0xFFu;
            const uint32_t size = tbl_s[L.model * DRA_MAX_PROFILES + prof] & 0xFFu;
            const uint32_t s_ = (uint32_t)((pos < 16u ? st_lo >> (4u * pos) : st_hi >> (4u * (pos - 16u))) & 0xFull);
            out[c.y] = make_uint2(g0 + gl, meta(s_, size, prof, DRA_ST_OK));
        }
    }
    return 0;
}

// thread per pod: validates the pod (spec §12: <= 32 claims, one node, slots inside out[]) and writes its record
//   {x = claims in the pod, y = node (0xFFFFFFFF: nothing to evaluate), z = first claim, w = 0}
// in the layout of a ClaimRec, so that the stable counting sort by node of the claim path orders the PODS by node.
// Malformed pods get their INVALID records here.
__global__ void __launch_bounds__(256)
k_pod_records(const uint4* __restrict__ claims, const uint32_t* __restrict__ pod_off, uint32_t n_pod, uint32_t n_node,
              const uint32_t* __restrict__ out_off, uint2* __restrict__ out, uint32_t n_out, uint4* __restrict__ podrec, Err err) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pod) return;
    const uint32_t c0 = __ldg(&pod_off[p]), c1 = __ldg(&pod_off[p + 1]);
    const uint32_t n = c1 - c0;
    uint4 rec = make_uint4(n, 0xFFFFFFFFu, c0, 0);
    if (n == 0 || c1 < c0) { podrec[p] = rec; return; }
    const bool have_off = out_off != nullptr;
    const uint32_t node = __ldg(&claims[c0]).y;
    bool bad = n > DRA_MAX_POD || node >= n_node, oor = false;
    for (uint32_t i = c0; i < c1; ++i) {
        const uint4 c = __ldg(&claims[i]);
        const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
        bad = bad || c.y != node;
        const uint32_t slots = (kind == DRA_KIND_GPU && c.y < n_node && !claim_invalid(kind, prof, count, have_off)) ? count : 1u;
        const uint32_t dst = have_off ? __ldg(&out_off[i]) : i;
        oor = oor || dst > n_out || slots > n_out - dst;
    }
    if (oor) { err.set(ERR_OUT_RANGE); podrec[p] = rec; return; }
    if (bad) {
        for (uint32_t i = c0; i < c1; ++i) {
            const uint4 c = __ldg(&claims[i]);
            const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
            const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : prof;
            const uint32_t slots = (kind == DRA_KIND_GPU && c.y < n_node && !claim_invalid(kind, prof, count, have_off)) ? count : 1u;
            const uint32_t dst = have_off ? __ldg(&out_off[i]) : i;
            for (uint32_t k = 0; k < slots; ++k) out[dst + k] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, DRA_ST_INVALID));
        }
        podrec[p] = rec; return;
    }
    rec.y = node;
    podrec[p] = rec;
}

struct PodArgs {
    const uint4* claims; const uint32_t* out_off; uint2* out;
    const uint4* sorted;          // pod records grouped by node (stable), output of the bucketing kernels
    const uint32_t* claim_off;    // [n_node+2] offsets into sorted
    const uint4* inv_src; uint4* inv_dst; const uint32_t* node_off; const uint32_t* tbl;
    uint32_t n_node, exhaustive; SelCtx sel; Err err;
};

// The placement table into the CTA's shared tbl_s, by its NT threads; every thread returns once it is in place
template <int NT>
__device__ __forceinline__ void stage_table(uint32_t* tbl_s, const uint32_t* tbl) {
    for (uint32_t i = threadIdx.x; i < DRA_MAX_MODELS * DRA_MAX_PROFILES; i += NT) tbl_s[i] = __ldg(&tbl[i]);
    __syncthreads();
}

// one warp per node, one lane per GPU; the node's pods in input order
template <int WPC>
__global__ void __launch_bounds__(WPC * 32)
k_pods(const PodArgs a) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    pdl_wait();
    stage_table<WPC * 32>(tbl_s, a.tbl);
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t node = blockIdx.x * WPC + wid; node < a.n_node; node += gridDim.x * WPC) {
        const uint32_t g0 = __ldg(&a.node_off[node]), ng = __ldg(&a.node_off[node + 1]) - g0;
        const uint32_t p0 = __ldcg(&a.claim_off[node]), p1 = __ldcg(&a.claim_off[node + 1]);
        uint4 rec = make_uint4(0, 0, 0, 0);
        if (lane < ng) rec = __ldg(&a.inv_src[g0 + lane]);
        Lane L; L.load(rec, lane < ng);
        for (uint32_t m = p0; m < p1; ++m) {
            const uint4 pr = __ldcg(&a.sorted[m]);
            const PodGet get{a.claims + pr.z, a.out_off ? a.out_off + pr.z : nullptr, pr.z};
            Lane Lt = L;
            (void)pod_eval<32>(Lt, lane, FULLMASK, 0, g0, tbl_s, get, pr.x, a.sel, a.exhaustive != 0, a.out_off != nullptr, a.out);
            L = Lt;
            __syncwarp();
        }
        if (lane < ng && (p1 > p0 || a.inv_src != a.inv_dst)) a.inv_dst[g0 + lane] = L.store(rec);
    }
}

// ====================================================================================================
// place pods (spec §13): pods in input order, each on the first candidate node where it fits on that node's current
// state — the classic controller's pending allocations (SURVEY App. A), applied to a whole batch in one pass
// ====================================================================================================
// Every node keeps a LIST of the visits the sequential rule can make to it, in the order it makes them (candidate form:
// the {pod, node, position} pair records, stably sorted by node; dense form: implicitly every pod at position = node),
// and a CURSOR into it.  Every pod keeps a state word: the position in its candidate list it has reached, a done bit and
// a "search budget ran out somewhere" bit.  One warp owns a node for the whole launch (one lane per GPU, as in k_pods);
// at entry (q, k) of its list it skips q when q is done or already past position k, evaluates q when q is AT k, and
// otherwise waits: q may still come here.  Exact: a node evaluates q only after every pod before q that lists the node
// has passed its cursor.  Progress: the lowest unfinished pod heads its current node's list (everything before it there
// belongs to finished pods or to its own earlier positions), so with every CTA resident the loop always advances.
constexpr uint32_t PL_DONE = 0x80000000u, PL_LIMIT = 0x40000000u, PL_POS = 0x3FFFFFFFu;

struct PlaceArgs {
    const uint4* claims; const uint32_t* pod_off; uint32_t n_pod;
    const uint32_t* cand_nodes; const uint32_t* cand_off;   // nullptr: dense form
    const uint32_t* out_off; uint2* out;
    uint32_t* state; uint32_t* pod_node;
    uint4* pairs;                 // candidate form: {pod, node (0xFFFFFFFF: never visited), position, 0} per candidate
    const uint4* sorted;          // the pairs stably sorted by node (the bucketing kernels), node n's at list_off[n] ..
    const uint32_t* list_off;
    uint32_t* cursor;             // [n_node] per node: entries of its list already passed; [n_node]: evaluations so far
    const uint4* inv_src; uint4* inv_dst; const uint32_t* node_off; const uint32_t* tbl;
    uint32_t n_node, exhaustive; SelCtx sel; Err err;
};

// Sharded form (dra_place_pods_batch_global_device): each rank walks the visit lists of its own node window, and every
// rank holds a REPLICA of every pod's state word.  A word is 64 bits, {call sequence : state}, and every publication is an
// atomic max into every rank's replica.  Within a call a pod's state only grows (positions rise, the limit bit is sticky,
// DONE is highest), and a word of an earlier call loses to any word of the current one, so a late or reordered delivery
// never moves a word back and nothing is ever reset.  The final word is DONE plus the global node the pod was placed on,
// or PL_NOWHERE.
constexpr uint32_t PL_NOWHERE = 0xFFFFFFFFu;
struct PlaceShard {
    unsigned long long* rep[PEER_MAX];   // rep[r]: rank r's replica of the state words (rep[rank]: this rank's own)
    uint32_t* prog[PEER_MAX];            // prog[r]: rank r's progress counter, +1 per publication anywhere, never reset
    const uint32_t* gated;               // the call words' SP_GATED: nothing is evaluated
    uint32_t* w;                         // the call words (SP_*): [r] slots rank r may finalise / finalises, SP_BAD
    uint4* podrec;                       // [n_pod] {claims, -, first claim, finalising rank or SP_NONE} for k_spod_gather
    uint32_t world, rank, seq;           // seq: this call's sequence number, the same on every rank
    uint32_t node_lo, n_win;             // this rank's node window [node_lo, node_lo + n_win)
    uint32_t n_claim, n_pair, n_out;     // what the device-side checks hold the arrays to
    uint32_t rank_hi[PEER_MAX];          // rank r serves nodes [rank_hi[r-1], rank_hi[r])
    long long spin_limit;                // cycles without a publication anywhere before ERR_PEER_TIMEOUT
};

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
    unsigned long long v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
    uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void red_max_release_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("red.release.sys.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// the rank whose node range holds global node n
__device__ __forceinline__ uint32_t place_owner(const PlaceShard& s, uint32_t n) {
    uint32_t o = 0;
    for (uint32_t q = 0; q + 1 < s.world; ++q) o += n >= s.rank_hi[q] ? 1u : 0u;
    return o;
}

// The final records of a pod placed nowhere (warp-wide): INVALID for the claims invalid by §3/§10 (every claim when the
// pod has more than 32), `st` for the others; slots counted as if each claim named a node of the inventory.
__device__ __forceinline__ void place_fail(const PlaceArgs& a, uint32_t c0, uint32_t cnt, uint32_t st, uint32_t lane) {
    const bool have_off = a.out_off != nullptr;
    for (uint32_t i = lane; i < cnt; i += 32) {
        const uint4 c = __ldg(&a.claims[c0 + i]);
        const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
        const bool shape = claim_invalid(kind, prof, count, have_off);
        const bool inv = cnt > DRA_MAX_POD || shape || claim_sel(kind, c.z, c.w) > a.sel.n_sel;
        const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : prof;
        const uint32_t slots = (kind == DRA_KIND_GPU && !shape) ? count : 1u;
        const uint32_t dst = have_off ? __ldg(&a.out_off[c0 + i]) : c0 + i;
        for (uint32_t k = 0; k < slots; ++k) a.out[dst + k] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, inv ? (uint32_t)DRA_ST_INVALID : st));
    }
}

// Warp per pod: the pod's state word (first usable position, or done), pod_node = NONE, the records of the pods that
// will never be evaluated (more than 32 claims, or no candidate naming a node of the inventory) and, candidate form, the
// pair records.  Pairs of pods that are never evaluated, and pairs naming no node, carry node NONE: the sort drops them.
__global__ void __launch_bounds__(256)
k_pods_place_prep(const PlaceArgs a) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p >= a.n_pod) return;
    const uint32_t c0 = __ldg(&a.pod_off[p]), cnt = __ldg(&a.pod_off[p + 1]) - c0;
    const bool live = cnt != 0 && cnt <= DRA_MAX_POD;
    uint32_t first = PL_DONE;
    if (!a.cand_off) {
        if (a.n_node) first = 0;
    } else {
        const uint32_t k0 = __ldg(&a.cand_off[p]), nk = __ldg(&a.cand_off[p + 1]) - k0;
        for (uint32_t j0 = 0; j0 < nk; j0 += 32) {
            const uint32_t j = j0 + lane;
            const uint32_t n = j < nk ? __ldg(&a.cand_nodes[k0 + j]) : 0xFFFFFFFFu;
            const bool usable = n < a.n_node;
            if (j < nk) a.pairs[k0 + j] = make_uint4(p, live && usable ? n : 0xFFFFFFFFu, j, 0);
            const uint32_t b = __ballot_sync(FULLMASK, usable);
            if (b && first == PL_DONE) first = j0 + (uint32_t)__ffs(b) - 1u;
        }
    }
    if (lane == 0) {
        a.pod_node[p] = DRA_GPU_NONE;
        a.state[p] = live ? first : PL_DONE;
    }
    if (cnt != 0 && (!live || first == PL_DONE)) place_fail(a, c0, cnt, live ? (uint32_t)DRA_ST_POD : (uint32_t)DRA_ST_INVALID, lane);
}

// Persistent: every CTA resident (cooperative launch); warp w owns nodes w, w + warps, ... and cycles over them.
// SHARD: the nodes are this rank's window (a.node_off, list_off and cursor are the window's; a.n_node is still the whole
// inventory, for the next usable candidate), states come from this rank's replica and go to every rank's, and warp 0
// stays until every pod's word here is DONE: a rank's own lists can end while pods still move on other ranks.  Launched
// without the cooperative attribute (cooperative grids do not run beside each other), sized to the rank's share of the
// residency.
template <int WPC, bool SHARD = false>
__global__ void __launch_bounds__(WPC * 32)
k_pods_place(const PlaceArgs a, const PlaceShard sh) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    if constexpr (SHARD) { if (__ldcg(sh.gated)) return; }
    stage_table<WPC * 32>(tbl_s, a.tbl);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t w0 = blockIdx.x * WPC + (threadIdx.x >> 5), n_warp = gridDim.x * WPC;
    const bool dense = a.cand_off == nullptr, have_off = a.out_off != nullptr;
    const uint32_t n_walk = SHARD ? sh.n_win : a.n_node, node_base = SHARD ? sh.node_lo : 0u;
    if (a.inv_src != a.inv_dst)                              // DRA_F_FRESH_INVENTORY: the owner copies its nodes first
        for (uint32_t node = w0; node < n_walk; node += n_warp) {
            const uint32_t g0 = __ldg(&a.node_off[node]), ng = __ldg(&a.node_off[node + 1]) - g0;
            if (lane < ng) a.inv_dst[g0 + lane] = __ldg(&a.inv_src[g0 + lane]);
        }
    uint32_t seen = 0;
    bool dead = false;
    long long t0 = clock64();
    while (true) {
        bool left = false, moved = false;
        for (uint32_t node = w0; node < n_walk; node += n_warp) {
            const uint32_t l0 = dense ? 0u : __ldcg(&a.list_off[node]), l1 = dense ? a.n_pod : __ldcg(&a.list_off[node + 1]);
            const uint32_t cur0 = l0 + __ldcg(&a.cursor[node]);
            uint32_t cur = cur0;
            if (cur >= l1) continue;
            const uint32_t g0 = __ldg(&a.node_off[node]), ng = __ldg(&a.node_off[node + 1]) - g0;
            Lane L;
            bool loaded = false, dirty = false;
            while (cur < l1) {
                // 32 entries at once: the first one that is not to be skipped
                const uint32_t e = cur + lane;
                uint32_t q = 0, k = 0, s = PL_DONE;
                if (e < l1) {
                    if (dense) { q = e; k = node + node_base; }
                    else { const uint4 r = __ldcg(&a.sorted[e]); q = r.x; k = r.z; }
                    if constexpr (SHARD) s = (uint32_t)ld_acquire_sys_u64(&sh.rep[sh.rank][q]);
                    else s = ld_acquire_u32(&a.state[q]);
                }
                const bool skip = (s & PL_DONE) || (s & PL_POS) > k;
                const uint32_t act = __ballot_sync(FULLMASK, !skip);
                if (!act) { cur = min(cur + 32u, l1); continue; }
                const uint32_t f = (uint32_t)__ffs(act) - 1u;
                cur += f;
                const uint32_t qf = __shfl_sync(FULLMASK, q, f), kf = __shfl_sync(FULLMASK, k, f), sf = __shfl_sync(FULLMASK, s, f);
                if ((sf & PL_POS) < kf) break;                   // q may still come here: this node waits
                if constexpr (SHARD) (void)ld_acquire_sys_u64(&sh.rep[sh.rank][qf]);
                else (void)ld_acquire_u32(&a.state[qf]);         // every lane: ordered after the previous owner's records
                if (!loaded) {
                    L.load(lane < ng ? a.inv_dst[g0 + lane] : make_uint4(0, 0, 0, 0), lane < ng);
                    loaded = true;
                }
                uint32_t st;
                {
                    const uint32_t c0 = __ldg(&a.pod_off[qf]), cnt = __ldg(&a.pod_off[qf + 1]) - c0;
                    const PodGet get{a.claims + c0, have_off ? a.out_off + c0 : nullptr, c0};
                    Lane Lt = L;
                    st = pod_eval<32>(Lt, lane, FULLMASK, 0, g0, tbl_s, get, cnt, a.sel, a.exhaustive != 0, have_off, a.out);
                    if (st == 0) L = Lt;
                }
                uint32_t next = PL_DONE;
                const uint32_t lim = (sf & PL_LIMIT) | (st == DRA_ST_SEARCH_LIMIT ? PL_LIMIT : 0u);
                if (st == 0) {
                    dirty = true;
                    if (!SHARD && lane == 0) a.pod_node[qf] = node;
                } else {
                    // the pod's next candidate that names a node of the inventory
                    if (dense) { if (kf + 1u < a.n_node) next = (kf + 1u) | lim; }
                    else {
                        const uint32_t k0 = __ldg(&a.cand_off[qf]), nk = __ldg(&a.cand_off[qf + 1]) - k0;
                        for (uint32_t j0 = kf + 1u; j0 < nk; j0 += 32) {
                            const uint32_t j = j0 + lane;
                            const bool usable = j < nk && __ldg(&a.cand_nodes[k0 + j]) < a.n_node;
                            const uint32_t b = __ballot_sync(FULLMASK, usable);
                            if (b) { next = (j0 + (uint32_t)__ffs(b) - 1u) | lim; break; }
                        }
                    }
                    if (next == PL_DONE) {
                        const uint32_t c0 = __ldg(&a.pod_off[qf]), cnt = __ldg(&a.pod_off[qf + 1]) - c0;
                        place_fail(a, c0, cnt, lim ? (uint32_t)DRA_ST_SEARCH_LIMIT : (uint32_t)DRA_ST_POD, lane);
                    }
                }
                if constexpr (SHARD) {
                    __threadfence_system();
                    __syncwarp();
                    if (lane == 0) {
                        const uint32_t wd = st == 0 ? (PL_DONE | (node + node_base)) : next == PL_DONE ? PL_NOWHERE : next;
                        const unsigned long long v = ((unsigned long long)sh.seq << 32) | wd;
                        for (uint32_t r = 0; r < sh.world; ++r) { red_max_release_sys_u64(sh.rep[r] + qf, v); red_add_sys_u32(sh.prog[r], 1u); }
                    }
                } else {
                    __threadfence();
                    __syncwarp();
                    if (lane == 0) { st_release_u32(&a.state[qf], next); atomicAdd(&a.cursor[a.n_node], 1u); }
                }
                moved = true;
                ++cur;
            }
            if (dirty && lane < ng) a.inv_dst[g0 + lane] = L.store(a.inv_dst[g0 + lane]);    // (only this warp writes the node)
            if (cur != cur0) { moved = true; a.cursor[node] = cur - l0; }     // (every lane: the next visit reads it on every lane)
            if (cur < l1) left = true;
        }
        if (!left) break;
        if (moved) { t0 = clock64(); continue; }
        // nothing moved on this warp's nodes: back off, and give up when no pod was evaluated anywhere for a long time
        // (cannot happen with every CTA resident; sharded: unless a peer stopped)
        __nanosleep(256);
        const uint32_t pr = __shfl_sync(FULLMASK, SHARD ? ld_acquire_sys_u32(sh.prog[sh.rank]) : ld_acquire_u32(&a.cursor[a.n_node]), 0);
        if (pr != seen) { seen = pr; t0 = clock64(); }
        else if (clock64() - t0 > (SHARD ? sh.spin_limit : 4000000000ll)) {
            if (lane == 0) a.err.set(SHARD ? ERR_PEER_TIMEOUT : ERR_DEVICE_WAIT);
            dead = true;
            break;
        }
    }
    if constexpr (SHARD) {
        if (w0 != 0 || dead) return;
        // every pod's word here DONE: then every evaluation of the call is over on every rank
        t0 = clock64();
        for (uint32_t p0 = 0; p0 < a.n_pod; ) {
            bool done = true;
            if (p0 + lane < a.n_pod) {
                const unsigned long long v = ld_acquire_sys_u64(&sh.rep[sh.rank][p0 + lane]);
                done = (uint32_t)(v >> 32) == sh.seq && ((uint32_t)v & PL_DONE);
            }
            if (__all_sync(FULLMASK, done)) { p0 += 32; continue; }
            __nanosleep(256);
            const uint32_t pr = __shfl_sync(FULLMASK, ld_acquire_sys_u32(sh.prog[sh.rank]), 0);
            if (pr != seen) { seen = pr; t0 = clock64(); }
            else if (clock64() - t0 > sh.spin_limit) { if (lane == 0) a.err.set(ERR_PEER_TIMEOUT); break; }
        }
    }
}

// ====================================================================================================
// UnsuitableNodes: warp per (pod, candidate) pair on a snapshot
// ====================================================================================================

struct UnsArgs {
    const uint4* claims; const uint32_t* pod_off; uint32_t n_pod;
    const uint32_t* cand_nodes; const uint32_t* cand_off; const uint32_t* pair_pod;   // cand_off == nullptr: dense form
    const uint4* inv; const uint32_t* node_off; uint32_t n_node; const uint32_t* tbl;
    uint32_t* bits;     // n_pair bits, zeroed by the caller, set with atomicOr
    SelCtx sel;
    uint32_t exhaustive; // spec §12: pod evaluation with the backtracking search
    unsigned long long* work;   // EXH: next unclaimed pair (zeroed by the caller) — searches differ by orders of magnitude
                                //      in length, so the warps take their pairs from a counter instead of a fixed stride
    uint32_t node_lo, n_win, n_walk;   // the node window (pair_decode; WIN = false: [0, n_node)), the pairs walked
    const uint32_t* gate;      // sharded call only: *gate != 0: the inputs failed their device-side check, evaluate nothing
};

struct GlobalGet {
    const uint4* base;
    __device__ __forceinline__ uint4 operator()(uint32_t m) const { return __ldg(&base[m]); }
};

// A counter walk's next G walk indices, for the whole warp: lane 0 takes them from the 64-bit counter (zeroed by the host)
// and every lane gets the first.  Every warp takes one value at or past the end, so the counter itself passes 2^32 on a
// walk near 2^32 pairs; the value is handed on clamped to 0xFFFFFFFF, which is at or past every walk's end.  A walk
// index below the end is a multiple of G below 2^32, so pw + grp never wraps.
template <uint32_t G>
__device__ __forceinline__ uint32_t walk_fetch(unsigned long long* work, uint32_t lane) {
    uint32_t nxt = 0;
    if (lane == 0) nxt = (uint32_t)min(atomicAdd(work, (unsigned long long)G), 0xFFFFFFFFull);
    return __shfl_sync(FULLMASK, nxt, 0);
}

// Walk index `walk` of a pair walk over the node window [node_lo, node_lo + n_win) as pod, node and pair.  Dense form (cand_off
// nullptr): walk w is pod w / n_win at node node_lo + w % n_win.  Candidate form: the walk index is the pair index.  False
// only for a candidate on another rank's node (of the inventory, outside the window); one naming no node is the caller's.
__device__ __forceinline__ bool pair_decode(uint32_t walk, uint32_t node_lo, uint32_t n_win, uint32_t n_node, const uint32_t* cand_off,
                                            const uint32_t* cand_nodes, const uint32_t* pair_pod, uint32_t& pod, uint32_t& node, uint32_t& pair) {
    if (!cand_off) { pod = walk / n_win; node = node_lo + (walk - pod * n_win); pair = pod * n_node + node; return true; }
    pair = walk; node = __ldg(&cand_nodes[pair]); pod = __ldg(&pair_pod[pair]);
    return !(node < n_node && node - node_lo >= n_win);
}

// Pod p's pairs [k0, k1): its candidates, or dense the columns [lo, lo + n_win) of its row.  T: the caller's index width.
template <class T>
__device__ __forceinline__ void pod_pairs(const uint32_t* cand_off, uint32_t p, uint32_t n_node, uint32_t lo, uint32_t n_win, T& k0, T& k1) {
    if (cand_off) { k0 = __ldg(&cand_off[p]); k1 = __ldg(&cand_off[p + 1]); } else { k0 = (T)p * n_node + lo; k1 = k0 + n_win; }
}

// The node of pod p's pair k: its candidate's node, or dense (cand_off nullptr) the pair's column
template <class T>
__device__ __forceinline__ uint32_t pair_node(const uint32_t* cand_off, const uint32_t* cand_nodes, T k, uint32_t p, uint32_t n_node) {
    return cand_off ? __ldg(&cand_nodes[k]) : (uint32_t)(k - (T)p * n_node);
}

// A lane of a pair kernel with W lanes per pair: lane gl of group grp, whose lanes are gbase .. gbase + W - 1 (gmask)
struct LaneGroup { uint32_t lane, grp, gl, gbase, gmask; };
template <int W>
__device__ __forceinline__ LaneGroup lane_group() {
    const uint32_t lane = threadIdx.x & 31, grp = lane / W, gbase = grp * W;
    return {lane, grp, lane - gbase, gbase, W == 32 ? FULLMASK : (((1u << (W & 31)) - 1u) << gbase)};
}

// W lanes per (pod, candidate) pair: 32/W pairs share a warp (W = 8 for the usual <= 8 GPUs per node), each
// group running its own claim loop with group-wide ballots.  Dense form: every pod against every node, no candidate arrays.
// WIN: the node window and the gate of the sharded call, else the window [0, n_node) (own instantiations: with the window
// the exhaustive kernel needs 81 registers instead of 78, which costs dra_unsuitable_batch a third of its CTAs per SM).
template <int WPC, int W, bool EXH, bool WIN>          // EXH: spec §12 (own instantiation: the default kernel stays as lean as it was)
__global__ void __launch_bounds__(WPC * 32, 2)
k_unsuitable(const UnsArgs a) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    if (WIN && a.gate && __ldcg(a.gate)) return;
    stage_table<WPC * 32>(tbl_s, a.tbl);
    constexpr uint32_t G = 32 / W;
    const auto [lane, grp, gl, gbase, gmask] = lane_group<W>();
    const uint32_t wid = threadIdx.x >> 5, stride = gridDim.x * WPC * G, n_walk = a.n_walk;
    const uint32_t node_lo = WIN ? a.node_lo : 0u, n_win = WIN ? a.n_win : a.n_node;
    // the stride steps at most to n_walk: a plain pw += stride wraps past 2^32 near the top of the range and walks again
    for (uint32_t pw = (blockIdx.x * WPC + wid) * G; ; pw += min(stride, n_walk - pw)) {
        if (EXH) pw = walk_fetch<G>(a.work, lane);
        if (pw >= n_walk) break;
        const uint32_t walk = pw + grp;
        if (walk >= n_walk) continue;                                    // whole group skips together
        uint32_t pod, node, pair;
        if (!pair_decode(walk, node_lo, n_win, a.n_node, a.cand_off, a.cand_nodes, a.pair_pod, pod, node, pair) ||
            node - node_lo >= n_win || pod >= a.n_pod) continue;         // another rank's node, or none: unsuitable here
        const uint32_t c0 = __ldg(&a.pod_off[pod]);
        const uint32_t cnt = __ldg(&a.pod_off[pod + 1]) - c0;
        const uint32_t g0 = __ldg(&a.node_off[node]);
        const uint32_t ng = __ldg(&a.node_off[node + 1]) - g0;
        uint4 rec = make_uint4(0, 0, 0, 0);
        if (gl < ng) rec = __ldg(&a.inv[g0 + gl]);
        Lane L; L.load(rec, gl < ng);
        if (EXH) {                                                        // spec §12
            if (cnt > DRA_MAX_POD || ng > W) continue;
            const PodGet pget{a.claims + c0, nullptr, 0};
            Lane Lt = L;                                                    // by copy: a reference would pin L in local memory
            const uint32_t st = pod_eval<W>(Lt, lane, gmask, gbase, g0, tbl_s, pget, cnt, a.sel, true, true, nullptr);
            if (st == 0 && gl == 0) atomicOr(&a.bits[pair >> 5], 1u << (pair & 31));
            continue;
        }
        Dead D; FlagSink sink; GlobalGet get{a.claims + c0};
        if (ng > W) sink.failed = true;                                   // cannot happen: W is chosen from the inventory
        uint32_t k = 0;
        while (k < cnt && !sink.stop()) k += node_step(L, D, lane, g0, tbl_s, get, k, cnt, sink, true, a.sel, gmask, gbase);
        if (!sink.failed && gl == 0) atomicOr(&a.bits[pair >> 5], 1u << (pair & 31));
    }
}

// ---- sharded UnsuitableNodes (dra_unsuitable_batch_global_device) ----------------------------------------------------
// Warp per pod: checks that pod_off (and cand_off) are monotone and span their arrays — every rank gets the same arrays,
// so every rank finds the same fault — and, in the candidate form, writes pair -> pod for the pod's candidates (the
// warp's lanes stride the pod's range: one pod with many candidates costs coalesced stores, not a serial loop).
// A fault sets ERR_BAD_OFFSETS, which gates k_unsuitable (UnsArgs::gate).
__global__ void __launch_bounds__(256)
k_uns_prep(const uint32_t* __restrict__ pod_off, const uint32_t* __restrict__ cand_off, uint32_t n_pod, uint32_t n_claim,
           uint32_t n_pair, uint32_t* __restrict__ pair_pod, Err err) {
    const uint32_t lane = threadIdx.x & 31, p = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (p == 0 && lane == 0) {
        const bool span = __ldg(&pod_off[0]) == 0 && __ldg(&pod_off[n_pod]) == n_claim &&
                          (!cand_off || (__ldg(&cand_off[0]) == 0 && __ldg(&cand_off[n_pod]) == n_pair));
        if (!span) err.set(ERR_BAD_OFFSETS);
    }
    if (p >= n_pod) return;
    bool bad = __ldg(&pod_off[p + 1]) < __ldg(&pod_off[p]);
    if (cand_off) {
        const uint32_t k0 = __ldg(&cand_off[p]), k1 = __ldg(&cand_off[p + 1]);
        bad = bad || k1 < k0 || k1 > n_pair;
        if (!bad) for (unsigned long long k = (unsigned long long)k0 + lane; k < k1; k += 32) pair_pod[k] = p;   // 64 bits: k1 may lie within 32 of 2^32
    }
    if (bad && lane == 0) err.set(ERR_BAD_OFFSETS);
}

// The bit exchange: the peer exchange (PeerExchange) with one slice per sender.  Latency matters little next to the
// evaluation (100 us to ms).  k_peer_push sends this rank's words (its own pairs' bits, every other bit zero; slices and
// the local words are padded to 16 bytes), then
//   k_uns_merge  block 0 raises this rank's flags (the push grid has completed, its stores are fenced); every block waits
//                for every peer's flag and ORs the world's slices into the caller's bytes, whatever the wait returned.  A
//                small grid of its own: ranks sharing one device must not find their evaluation's SMs held by a peer's
//                waiting CTAs.
// A rank is never two calls ahead, since its next merge waits for this rank's next push.  With world 1 (an all-zero
// PeerExchange: no peers) the merge only turns the words into ceil(n_pair/8) bytes.
struct UnsMerge {
    const uint32_t* bits;         // this rank's words
    uint8_t* out;                 // ceil(n_pair / 8) bytes
    uint32_t n_words, n_bytes;
    uint32_t stride;              // words of one sender's slice: sender s's at PeerExchange::my_stage + s * stride words
};

__global__ void __launch_bounds__(256)
k_uns_merge(const PeerExchange x, const UnsMerge m) {
    const uint32_t tid = threadIdx.x;
    if (blockIdx.x == 0) peer_raise(x, tid);
    peer_wait(x, tid, clock64());
    __syncthreads();
    const uint32_t* my_stage = reinterpret_cast<const uint32_t*>(x.my_stage);
    const uint32_t world = x.world, rank = x.rank;           // (read from the parameters once: 32 registers, not 34)
    const bool whole = (reinterpret_cast<uintptr_t>(m.out) & 3u) == 0;
    for (uint32_t w = blockIdx.x * blockDim.x + tid; w < m.n_words; w += gridDim.x * blockDim.x) {
        uint32_t v = __ldcg(&m.bits[w]);
        for (uint32_t s = 0; s < world; ++s)
            if (s != rank) v |= __ldcg(&my_stage[(size_t)s * m.stride + w]);
        const uint32_t b0 = w * 4;
        if (whole && b0 + 4 <= m.n_bytes) *reinterpret_cast<uint32_t*>(m.out + b0) = v;
        else for (uint32_t b = 0; b < 4 && b0 + b < m.n_bytes; ++b) m.out[b0 + b] = (uint8_t)(v >> (8 * b));
    }
}

// The inventory sync (dra_shard_sync_inventory_device): every rank's GPU records of its own range to every peer, so that
// every live copy becomes the world's state, over the peer exchange (PeerExchange).  Owned ranges are disjoint, so every
// rank writes its records at their GLOBAL indices into one staging area per peer: k_peer_push sends this rank's GPUs
// [own_lo, own_hi) of the live copy, then
//   k_isync_copy  a grid of at most SMs / 4 CTAs.  The first CTA to arrive (one atomicMax on `elect`) raises this rank's
//                 flags, waits for every peer's flag and publishes ONE verdict for the call in `elect`; the other CTAs wait
//                 for that verdict (locally) and all of them copy GPUs outside [own_lo, own_hi) from staging into the live
//                 copy only when every peer arrived.  One verdict makes it all or nothing: a timed-out call leaves the live
//                 copy as it was.  The elected CTA started before any CTA waiting for it, so those wait at most twice the
//                 spin limit.
// A rank is never two calls ahead, since its next copy kernel waits for this rank's next flag, which this rank raises only
// after its copy of the call before.
struct InvSync {
    uint4* inv;                   // the live copy
    uint32_t* elect;              // [0] the last call whose CTA was elected, [1] that call's verdict: seq << 1 | all arrived
    uint32_t n_gpu, own_lo, own_hi;
};

__global__ void __launch_bounds__(256)
k_isync_copy(const PeerExchange x, const InvSync s) {
    __shared__ uint32_t s_lead, s_ok;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) { s_lead = atomicMax(&s.elect[0], x.seq) < x.seq; s_ok = 1u; }
    __syncthreads();
    const long long t0 = clock64();
    if (s_lead) {
        peer_raise(x, tid);
        if (!peer_wait(x, tid, t0)) s_ok = 0u;
        __syncthreads();
        if (tid == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(s.elect + 1), "r"(x.seq << 1 | s_ok) : "memory");
    } else {
        if (tid == 0) {
            uint32_t v;
            do {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(s.elect + 1) : "memory");
                if ((v >> 1) == (x.seq & 0x7FFFFFFFu)) { s_ok = v & 1u; break; }
                if (clock64() - t0 > 2 * x.spin_limit) { x.err.set(ERR_PEER_TIMEOUT); s_ok = 0u; break; }
            } while (true);
        }
        __syncthreads();
    }
    if (!s_ok) return;
    for (uint32_t i = blockIdx.x * blockDim.x + tid; i < s.n_gpu; i += gridDim.x * blockDim.x)
        if (i < s.own_lo || i >= s.own_hi) s.inv[i] = __ldcg(&x.my_stage[i]);
}

// ====================================================================================================
// Deallocate: thread per claim, atomics on the GpuRec words (updates commute, spec §9)
// ====================================================================================================
// slots(c) exactly as Allocate counted them (spec §9): an INVALID claim — here: one naming no node — has one
__device__ __forceinline__ uint32_t dealloc_slots(const uint4 c, uint32_t n_node, bool have_off) {
    const uint32_t kind = c.x & 0xFFu, count = c.x >> 16;
    return (kind == DRA_KIND_GPU && c.y < n_node && count >= 1 && count <= DRA_MAX_COUNT && (have_off || count == 1)) ? count : 1u;
}

// The slices an OutRec's u8 start and size name (spec §9): ((1 << size) - 1) << start cut to 16 bits, empty when start >= 16.
// Written without a shift of 32 or more, so the answer does not rest on how the hardware treats such counts.
__device__ __forceinline__ uint32_t slice_mask(const uint32_t start, const uint32_t size) {
    return start >= 16u ? 0u : (((size >= 16u ? 0xFFFFu : (1u << size) - 1u) << start) & 0xFFFFu);
}

// The sharded Deallocate's all-or-nothing check (dra_deallocate_batch_global_device), grid-stride over every claim: a slot
// range [base, base + slots) outside [0, n_out) sets ERR_BAD_DEALLOC, which gates k_dealloc.  Every rank reads the same
// arrays, so every rank finds the same fault.
__global__ void __launch_bounds__(256)
k_dealloc_check(const uint4* __restrict__ claims, uint32_t n_claim, const uint32_t* __restrict__ out_off, uint32_t n_out,
                uint32_t n_node, Err err) {
    pdl_trigger();                                          // k_dealloc may be scheduled now; it waits for this grid
    const bool have_off = out_off != nullptr;
    bool bad = false;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_claim; i += gridDim.x * blockDim.x) {
        const uint32_t base = have_off ? __ldg(&out_off[i]) : i, slots = dealloc_slots(__ldg(&claims[i]), n_node, have_off);
        bad = bad || base > n_out || slots > n_out - base;
    }
    if (bad) err.set(ERR_BAD_DEALLOC);
}

// GPUs outside [gpu_lo, gpu_hi) are not written (dra_deallocate_batch: [0, n_gpu)).  gate: when set (the sharded call,
// launched as a programmatic dependent of k_dealloc_check), a non-zero word means the check found a bad slot range and
// nothing is applied.  dra_deallocate_batch checks every slot range on the host before it launches, so the ERR_OUT_RANGE
// test below only guards a launch that skipped that check.
__global__ void __launch_bounds__(256)
k_dealloc(const uint4* __restrict__ claims, uint32_t n_claim, const uint32_t* __restrict__ out_off,
          const uint2* __restrict__ out, uint32_t n_out, uint32_t* __restrict__ inv, uint32_t gpu_lo, uint32_t gpu_hi,
          uint32_t n_node, const uint32_t* gate, Err err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_claim) return;
    const uint4 c = __ldg(&claims[i]);
    const uint32_t kind = c.x & 0xFFu;
    const bool have_off = out_off != nullptr;
    const uint32_t base = have_off ? __ldg(&out_off[i]) : i;
    const uint32_t slots = dealloc_slots(c, n_node, have_off);
    if (gate) {
        pdl_wait();                                         // the check's grid has completed and its gate word is visible
        if (*(volatile const uint32_t*)gate) return;
    }
    if (base > n_out || slots > n_out - base) { err.set(ERR_OUT_RANGE); return; }
    for (uint32_t s = 0; s < slots; ++s) {
        const uint2 o = __ldg(&out[base + s]);
        if ((o.y >> 24) != DRA_ST_OK || o.x < gpu_lo || o.x >= gpu_hi) continue;
        uint32_t* w = inv + (size_t)o.x * 4;
        if (kind == DRA_KIND_GPU) atomicAnd(&w[0], ~((uint32_t)DRA_GPU_FULL_ALLOCATED << 16));
        else if (kind == DRA_KIND_MIG) atomicAnd(&w[0], ~slice_mask(o.y & 0xFFu, (o.y >> 8) & 0xFFu));
        else if (kind == DRA_KIND_SHARED) {
            atomicAdd(&w[1], c.z);
            uint32_t old = w[3], assumed;
            do { assumed = old; old = atomicCAS(&w[3], assumed, (assumed & 0xFFFF0000u) | ((assumed - 1u) & 0xFFFFu)); }
            while (old != assumed);
        }
    }
}


// ====================================================================================================
// the all-gather as its own kernel (sort path: the pack kernel has no tail), same packets as k_fused's tail
// ====================================================================================================
// Warp-collective: one reservation per warp of the lanes' n packets, contiguous in this rank's slice, so that they leave
// as 128-byte lines on the wire.  Returns the lane's first position.
__device__ __forceinline__ uint32_t pkt_warp_reserve(const PktGather& g, uint32_t n) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t incl = n;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULLMASK, incl, d); if (lane >= (uint32_t)d) incl += y; }
    const uint32_t tot = __shfl_sync(FULLMASK, incl, 31);
    uint32_t base = 0;
    if (lane == 0 && tot) base = atomicAdd(&g.cursor[g.parity], tot);
    return __shfl_sync(FULLMASK, base, 0) + incl - n;
}

// claims[0..n) are THIS rank's claims (input order or sorted, any order), out_off their first local slot (NULL: slot i);
// their OutRecs already sit in the local table at slot_base + slot.  Thread per claim: send; then everybody receives.
__global__ void __launch_bounds__(256)
k_pkt_gather(const PktGather g, const uint4* __restrict__ claims, uint32_t n_claim, const uint32_t* __restrict__ n_dev,
             const uint32_t* __restrict__ out_off, uint32_t n_out, uint32_t have_off, uint32_t n_node, Err err) {
    const uint32_t T = blockIdx.x * blockDim.x + threadIdx.x, NT = gridDim.x * blockDim.x;
    if (n_dev) n_claim = min(n_claim, __ldcg(n_dev));
    if (blockIdx.x == 0 && threadIdx.x == 32) g.cursor[g.parity ^ 1u] = 0;
    const uint2* local = g.table + g.slot_base;
    for (uint32_t i0 = blockIdx.x * blockDim.x; i0 < n_claim; i0 += NT) {
        const uint32_t i = i0 + threadIdx.x;
        uint32_t sl = 0, dst = 0;
        if (i < n_claim) {
            const uint4 c = __ldcg(&claims[i]);
            const uint32_t kind = c.x & 0xFFu, count = c.x >> 16;
            dst = out_off ? __ldcg(&out_off[i]) : i;
            sl = (kind == DRA_KIND_GPU && c.y < n_node && !claim_invalid(kind, 0, count, have_off != 0)) ? count : 1u;
            if (dst > n_out || sl > n_out - dst) sl = 0;
        }
        const uint32_t base = pkt_warp_reserve(g, sl);
        for (uint32_t s_ = 0; s_ < sl; ++s_)
            if (base + s_ < g.cap) pkt_send(g, base + s_, __ldcg(local + dst + s_), g.slot_base + dst + s_);
    }
    pkt_finish_send(g);
    pkt_receive(g, T, NT, err);
}

// ====================================================================================================
// sharded pods Allocate (dra_allocate_pods_batch_global_device): every rank reads the WHOLE pod array
// ====================================================================================================
// A non-empty pod belongs to the rank whose node range holds its FIRST claim's node (a node outside the inventory: the
// stray rank).  Every rank validates every pod on GLOBAL node indices and counts every rank's slots (the gather's expected
// counts); the owner writes the INVALID records of its malformed pods and keys its well-formed pods by their node inside
// its window for the claim path's counting sort (any other pod gets no node, and the sort drops it — the sort is stable,
// so a node's pods stay in input order).  k_pods then runs unchanged on the window.
// Call words (SPodArgs::w), zeroed by the host before the call up to and including SP_BAD:
constexpr uint32_t SP_BAD = PEER_MAX;             // a fault in the inputs (every rank finds the same one)
constexpr uint32_t SP_EXPECT = 2 * PEER_MAX;      // [PEER_MAX] packets expected from each rank (its slots, at least 1)
constexpr uint32_t SP_NDEV = 3 * PEER_MAX;        // pod records the sort takes: n_pod, or 0 when the call is gated
constexpr uint32_t SP_GATED = 3 * PEER_MAX + 1;   // nothing is evaluated or sent
constexpr uint32_t SP_WORDS = 4 * PEER_MAX;
constexpr uint32_t SP_NONE = 0xFFFFFFFFu;
struct SPodArgs {
    const uint4* claims; const uint32_t* pod_off; const uint32_t* out_off;
    uint32_t n_claim, n_pod, n_out, n_node;       // n_node: the whole inventory
    uint32_t node_lo, node_hi, take_stray;        // this rank's window; take_stray: it owns pods naming no node
    uint32_t rank, world, stray_rank;             // world > 1: counted with rank_hi (the shard map)
    uint32_t rank_hi[PEER_MAX];                   // rank r serves nodes [rank_hi[r-1], rank_hi[r])
    uint2* table;                                 // this rank's table, global slots
    uint4* podrec;                                // [n_pod] {claims, window node or SP_NONE, first claim, owner rank or SP_NONE}
    uint32_t* w;                                  // [SP_WORDS] call words
    Err err;
};

// OutRec slots of one claim of a pod (spec §1/§3): `count` for a well-formed GPU claim naming a node of the inventory, else 1
__device__ __forceinline__ uint32_t pod_claim_slots(const uint4 c, uint32_t n_node, bool have_off) {
    const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
    return (kind == DRA_KIND_GPU && c.y < n_node && !claim_invalid(kind, prof, count, have_off)) ? count : 1u;
}
// ... and as place pods counts them (spec §13): as if the claim named a node of the inventory, whatever its node field
__device__ __forceinline__ uint32_t place_claim_slots(const uint4 c, bool have_off) {
    const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
    return (kind == DRA_KIND_GPU && !claim_invalid(kind, prof, count, have_off)) ? count : 1u;
}

// thread per pod, every pod: the checks of k_pod_records plus the device-side ones (pod_off monotone and spanning
// [0, n_claim]) — those set SP_BAD instead of failing one pod, since every rank sees the same arrays
__global__ void __launch_bounds__(256)
k_spod_records(const SPodArgs a) {
    __shared__ uint32_t rs_s[PEER_MAX];
    const uint32_t tid = threadIdx.x, p = blockIdx.x * blockDim.x + tid;
    if (tid < PEER_MAX) rs_s[tid] = 0;
    __syncthreads();
    if (p < a.n_pod) {
        const uint32_t c0 = __ldg(&a.pod_off[p]), c1 = __ldg(&a.pod_off[p + 1]);
        uint4 rec = make_uint4(c1 - c0, SP_NONE, c0, SP_NONE);
        bool fault = p == 0 && (c0 != 0 || __ldg(&a.pod_off[a.n_pod]) != a.n_claim);
        if (c1 < c0 || c1 > a.n_claim) fault = true;
        else if (c1 > c0) {
            const bool have_off = a.out_off != nullptr;
            const uint32_t node = __ldg(&a.claims[c0]).y;
            bool bad = c1 - c0 > DRA_MAX_POD || node >= a.n_node;
            uint32_t total = 0;
            for (uint32_t i = c0; i < c1; ++i) {
                const uint4 c = __ldg(&a.claims[i]);
                bad = bad || c.y != node;
                const uint32_t slots = pod_claim_slots(c, a.n_node, have_off);
                const uint32_t dst = have_off ? __ldg(&a.out_off[i]) : i;
                fault = fault || dst > a.n_out || slots > a.n_out - dst;
                total += slots;
            }
            const bool stray = node >= a.n_node;
            const bool mine = stray ? a.take_stray != 0 : (node >= a.node_lo && node < a.node_hi);
            if (!fault) {
                if (a.world > 1) {
                    uint32_t o = a.stray_rank;
                    if (!stray) { o = 0; for (uint32_t q = 0; q + 1 < a.world; ++q) o += node >= a.rank_hi[q] ? 1u : 0u; }
                    atomicAdd(&rs_s[o], total);
                }
                if (mine) {
                    rec.w = a.rank;
                    if (!bad) rec.y = node - a.node_lo;
                    else for (uint32_t i = c0; i < c1; ++i) {
                        const uint4 c = __ldg(&a.claims[i]);
                        const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu;
                        const uint32_t op = kind == DRA_KIND_GPU ? DRA_PROFILE_GPU : kind == DRA_KIND_SHARED ? DRA_PROFILE_SHARED : prof;
                        const uint32_t slots = pod_claim_slots(c, a.n_node, have_off);
                        const uint32_t dst = have_off ? __ldg(&a.out_off[i]) : i;
                        for (uint32_t k = 0; k < slots; ++k) a.table[dst + k] = make_uint2(DRA_GPU_NONE, meta(0, 0, op, DRA_ST_INVALID));
                    }
                }
            }
        }
        if (fault) { a.w[SP_BAD] = 1u; a.err.set(ERR_BAD_PODS); }
        a.podrec[p] = rec;
    }
    __syncthreads();
    if (a.world > 1 && tid < a.world && rs_s[tid]) atomicAdd(&a.w[tid], rs_s[tid]);
}

// After the records, before the sort: decides whether the call goes ahead (no fault, and every rank's packets fit the
// staging slices: cap), publishes the sort's record count and the gather's expected counts, and — DRA_F_FRESH_INVENTORY
// (inv_src = the pristine copy) — copies this rank's GPUs from the pristine copy to the live one, so that k_pods reads and
// writes the live copy alone.  A gated call changes no inventory.  Every block decides alike; block 0 publishes.
__global__ void __launch_bounds__(256)
k_spod_gate(const SPodArgs a, uint32_t cap, const uint4* __restrict__ inv_src, uint4* __restrict__ inv_dst,
            const uint32_t* __restrict__ node_off) {
    const uint32_t tid = threadIdx.x;
    const bool over = a.world > 1 && tid < a.world && __ldcg(&a.w[tid]) > cap;
    const bool gated = __syncthreads_or(over || __ldcg(&a.w[SP_BAD]) != 0) != 0;
    if (blockIdx.x == 0) {
        if (tid < PEER_MAX) a.w[SP_EXPECT + tid] = gated ? 1u : max(__ldcg(&a.w[tid]), 1u);
        if (tid == 0) { a.w[SP_NDEV] = gated ? 0u : a.n_pod; a.w[SP_GATED] = gated ? 1u : 0u; }
        if (over) a.err.set(ERR_BAD_PODS);
    }
    if (gated || !inv_src) return;
    const uint32_t g1 = __ldg(&node_off[a.node_hi]);
    for (uint32_t i = __ldg(&node_off[a.node_lo]) + blockIdx.x * blockDim.x + tid; i < g1; i += gridDim.x * blockDim.x)
        inv_dst[i] = __ldg(&inv_src[i]);
}

// The all-gather of the owned pods' records, with the packets of k_pkt_gather (global slots, expected counts known from
// k_spod_records, so no header).  Thread per pod; a pod's slots need not be contiguous, the slot rides in the packet.
// A rank with nothing to send — it owns no slot, or the call is gated — sends one packet addressed to the table's padding
// slot pad_slot instead (k_spod_gate expects it): each call is then a real exchange with every peer, so no rank gets two
// calls ahead of a peer still reading the staging slices of the same parity.
// ANY_NODE (sharded place pods): a claim's node field is ignored, slots are counted as if it named a node (spec §13).
template <bool ANY_NODE = false>
__global__ void __launch_bounds__(256)
k_spod_gather(const PktGather g, const SPodArgs a, uint32_t pad_slot) {
    const uint32_t T = blockIdx.x * blockDim.x + threadIdx.x, NT = gridDim.x * blockDim.x;
    if (blockIdx.x == 0 && threadIdx.x == 32) g.cursor[g.parity ^ 1u] = 0;
    const bool gated = __ldcg(&a.w[SP_GATED]) != 0;
    if (T == 0 && (gated || __ldcg(&a.w[g.rank]) == 0)) pkt_send(g, atomicAdd(&g.cursor[g.parity], 1u), make_uint2(0u, 0u), pad_slot);
    const uint32_t n_pod = gated ? 0u : a.n_pod;
    const bool have_off = a.out_off != nullptr;
    for (uint32_t p0 = blockIdx.x * blockDim.x; p0 < n_pod; p0 += NT) {
        const uint32_t p = p0 + threadIdx.x;
        uint4 rec = make_uint4(0u, SP_NONE, 0u, SP_NONE);
        if (p < n_pod) rec = __ldcg(&a.podrec[p]);
        const bool mine = rec.w == g.rank;
        auto slots = [&](uint32_t i) {
            const uint4 c = __ldg(&a.claims[i]);
            return ANY_NODE ? place_claim_slots(c, have_off) : pod_claim_slots(c, a.n_node, have_off);
        };
        uint32_t sl = 0;
        if (mine) for (uint32_t i = rec.z; i < rec.z + rec.x; ++i) sl += slots(i);
        uint32_t pos = pkt_warp_reserve(g, sl);
        if (!mine) continue;
        for (uint32_t i = rec.z; i < rec.z + rec.x; ++i) {
            const uint32_t s = slots(i);
            const uint32_t dst = have_off ? __ldg(&a.out_off[i]) : i;
            for (uint32_t k = 0; k < s; ++k, ++pos)
                if (pos < g.cap) pkt_send(g, pos, __ldcg(&g.table[dst + k]), dst + k);
        }
    }
    pkt_receive(g, T, NT, a.err);
}

// ====================================================================================================
// sharded place pods (dra_place_pods_batch_global_device): every rank reads the WHOLE pod and candidate arrays
// ====================================================================================================
// k_splace_prep -> k_spod_gate -> counting sort of the pairs on the window -> k_pods_place<4, true> -> k_splace_final ->
// k_spod_gate (expected counts) -> k_spod_gather<true>.  The call words are SPodArgs' (zeroed by the host up to SP_BAD).

// Warp per pod, every pod: the device-side checks (pod_off and cand_off monotone and spanning their arrays, at most PL_POS
// candidates, slots inside n_out — a fault sets SP_BAD and the pod writes nothing); the pod's initial state word, maxed into
// this rank's replica (a peer may already have moved it further in this call); the pair records keyed by WINDOW node (a
// candidate on another rank's node, or naming no node, gets none and the sort drops it); the final records of the pods that
// are never evaluated, which every rank writes alike into its own table; and, world > 1, the slots of every pod that has a
// usable candidate in rank r's range added to w[r] — an upper bound of what r can finalise, checked against the packet room
// by k_spod_gate before anything is placed.
__global__ void __launch_bounds__(256)
k_splace_prep(const PlaceArgs a, const PlaceShard sh) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p >= a.n_pod) return;
    const bool dense = a.cand_off == nullptr, have_off = a.out_off != nullptr;
    const uint32_t c0 = __ldg(&a.pod_off[p]), c1 = __ldg(&a.pod_off[p + 1]);
    bool fault = c1 < c0 || c1 > sh.n_claim || (p == 0 && (c0 != 0 || __ldg(&a.pod_off[a.n_pod]) != sh.n_claim));
    uint32_t k0 = 0, nk = 0;
    if (!dense) {
        const uint32_t k1 = __ldg(&a.cand_off[p + 1]);
        k0 = __ldg(&a.cand_off[p]);
        fault = fault || k1 < k0 || k1 > sh.n_pair || k1 - k0 > PL_POS || (p == 0 && (k0 != 0 || __ldg(&a.cand_off[a.n_pod]) != sh.n_pair));
        nk = k1 - k0;
    }
    uint32_t total = 0;
    if (!fault)
        for (uint32_t i = c0 + lane; i < c1; i += 32) {
            const uint32_t slots = place_claim_slots(__ldg(&a.claims[i]), have_off), dst = have_off ? __ldg(&a.out_off[i]) : i;
            fault = fault || dst > sh.n_out || slots > sh.n_out - dst;
            total += slots;
        }
    if (__any_sync(FULLMASK, fault)) {
        if (lane == 0) { sh.w[SP_BAD] = 1u; a.err.set(ERR_BAD_PODS); }
        return;
    }
    total = __reduce_add_sync(FULLMASK, total);
    const uint32_t cnt = c1 - c0;
    const bool live = cnt != 0 && cnt <= DRA_MAX_POD;
    uint32_t first = PL_DONE, owners = 0;
    if (dense) {
        if (a.n_node) first = 0;
        if (lane < sh.world && (lane ? sh.rank_hi[lane - 1] : 0u) < sh.rank_hi[lane]) owners = 1u << lane;
    } else {
        for (uint32_t j0 = 0; j0 < nk; j0 += 32) {
            const uint32_t j = j0 + lane;
            const uint32_t n = j < nk ? __ldg(&a.cand_nodes[k0 + j]) : 0xFFFFFFFFu;
            const bool usable = n < a.n_node;
            if (j < nk) a.pairs[k0 + j] = make_uint4(p, live && usable && n - sh.node_lo < sh.n_win ? n - sh.node_lo : 0xFFFFFFFFu, j, 0);
            const uint32_t b = __ballot_sync(FULLMASK, usable);
            if (b && first == PL_DONE) first = j0 + (uint32_t)__ffs(b) - 1u;
            if (usable) owners |= 1u << place_owner(sh, n);
        }
    }
    owners = __reduce_or_sync(FULLMASK, owners);
    const bool walks = live && first != PL_DONE;
    if (lane == 0) atomicMax(&sh.rep[sh.rank][p], ((unsigned long long)sh.seq << 32) | (walks ? first : PL_NOWHERE));
    if (cnt != 0 && !walks) place_fail(a, c0, cnt, live ? (uint32_t)DRA_ST_POD : (uint32_t)DRA_ST_INVALID, lane);
    if (walks && sh.world > 1 && lane < sh.world && ((owners >> lane) & 1u)) atomicAdd(&sh.w[lane], total);
}

// Thread per pod, after the walk (every word here is DONE): pod_node from the final word, and the pod's FINALISER — the
// rank that wrote its final records: the owner of the node it was placed on; placed nowhere, the owner of its last usable
// candidate (its last evaluation); never evaluated, none (every rank wrote those).  podrec and, world > 1, every
// finaliser's slots in w[r] (zeroed by the host after the first gate): the packets k_spod_gather sends and expects.
__global__ void __launch_bounds__(256)
k_splace_final(const PlaceArgs a, const PlaceShard sh) {
    __shared__ uint32_t rs_s[PEER_MAX];
    const uint32_t tid = threadIdx.x, p = blockIdx.x * blockDim.x + tid;
    if (tid < PEER_MAX) rs_s[tid] = 0;
    __syncthreads();
    if (p < a.n_pod) {
        const bool gated = __ldcg(sh.gated) != 0;
        uint32_t node = DRA_GPU_NONE, fin = SP_NONE, c0 = 0, cnt = 0;
        if (!gated) {
            c0 = __ldg(&a.pod_off[p]); cnt = __ldg(&a.pod_off[p + 1]) - c0;
            const unsigned long long v = __ldcg(&sh.rep[sh.rank][p]);
            const uint32_t wd = (uint32_t)v;
            const bool final_ = (uint32_t)(v >> 32) == sh.seq && (wd & PL_DONE);    // (not after ERR_PEER_TIMEOUT)
            if (final_ && (wd & ~PL_DONE) < a.n_node) { node = wd & ~PL_DONE; fin = place_owner(sh, node); }
            else if (final_ && cnt != 0 && cnt <= DRA_MAX_POD) {
                if (!a.cand_off) { if (a.n_node) fin = place_owner(sh, a.n_node - 1); }
                else
                    for (uint32_t j = __ldg(&a.cand_off[p + 1]), k0 = __ldg(&a.cand_off[p]); j > k0; --j) {
                        const uint32_t n = __ldg(&a.cand_nodes[j - 1]);
                        if (n < a.n_node) { fin = place_owner(sh, n); break; }
                    }
            }
            if (fin != SP_NONE && sh.world > 1) {
                uint32_t total = 0;
                for (uint32_t i = c0; i < c0 + cnt; ++i) total += place_claim_slots(__ldg(&a.claims[i]), a.out_off != nullptr);
                atomicAdd(&rs_s[fin], total);
            }
        }
        a.pod_node[p] = node;
        sh.podrec[p] = make_uint4(cnt, SP_NONE, c0, fin);
    }
    __syncthreads();
    if (sh.world > 1 && tid < sh.world && rs_s[tid]) atomicAdd(&sh.w[tid], rs_s[tid]);
}

// ====================================================================================================
// adjacent integer searches of the reference, batched (SURVEY §8f-4; API completeness)
// ====================================================================================================
// limit.Megabyte() — api/nvidia.com/resource/gpu/v1alpha1/sharing.go:234-237: v = bytes/1024/1024 truncated toward
// zero (Go and C agree), valid iff v > 0.
__global__ void __launch_bounds__(256)
k_mps_limits(const long long* __restrict__ bytes, uint32_t n, long long* __restrict__ mib, uint8_t* __restrict__ valid) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long v = bytes[i] / 1024 / 1024;
    mib[i] = v; valid[i] = v > 0 ? 1 : 0;
}

// imexDomainOffsets.add's search — cmd/nvidia-dra-controller/imex.go:336-349: lowest multiple of `step` below
// `limit` that is not in the domain's used list; -1 = "channel limit reached".  One warp per domain, lane = candidate
// window (limit/step <= 32 in the reference: 2048/128 = 16); wider ranges loop.
__global__ void __launch_bounds__(256)
k_imex_offsets(const int* __restrict__ used, const uint32_t* __restrict__ dom_off, uint32_t n_dom, int step, int limit,
               int* __restrict__ out) {
    const uint32_t lane = threadIdx.x & 31, dom = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (dom >= n_dom) return;
    const uint32_t u0 = dom_off[dom], u1 = dom_off[dom + 1];
    int found = -1;
    for (int base = 0; base < limit && found < 0; base += 32 * step) {
        const int off = base + (int)lane * step;
        bool taken = off >= limit;
        for (uint32_t k = u0; k < u1 && !taken; ++k) taken = used[k] == off;
        const uint32_t freeb = __ballot_sync(FULLMASK, !taken);
        if (freeb) found = base + ((int)__ffs(freeb) - 1) * step;
    }
    if (lane == 0) out[dom] = found;
}

// ====================================================================================================
// Preemption (spec §14): per (pending pod, candidate node) pair, which lower-priority running pods to evict — remove every
// one of them, then reprieve them from the most important down (kube-scheduler's SelectVictimsOnNode) — and per pod the
// node to evict them on (pickOneNodeForPreemption).  Pure: the inventory is read, never written.
//   k_pre_running   thread per running pod: checks its offsets and slots, finds its node, writes its record
//   (bucketing)     the records grouped by node with the stable counting sort of the claim path
//   k_pre_vsort     CTA per node: the node's list by priority descending, index ascending (rank by counting)
//   k_pods_preempt  W lanes per pair, one per GPU of the node: dry pod_eval, remove V, pod_eval, the reprieve loop
//   k_pre_choose    warp per pod: the pod's pairs reduced in list order
//   k_pods_preempt_victims  W lanes per pod: the reprieve of the chosen pair again, this time writing the victims
// The sharded call (below) runs the same two pair kernels on its rank's node window.
// ====================================================================================================
struct PreArgs {
    const uint4* claims; const uint32_t* pod_off; const int32_t* prio; uint32_t n_pod;
    const uint32_t* cand_nodes; const uint32_t* cand_off; const uint32_t* pair_pod;   // cand_off == nullptr: dense form
    uint32_t n_pair;
    const uint4* rclaims; uint32_t rn_claim; const uint32_t* rpod_off; const int32_t* rprio; uint32_t rn_pod;
    const uint32_t* rout_off; const uint2* rout; uint32_t rn_out;
    uint4* rrec;                  // [rn_pod] {claims, node or NONE, first claim, prio}: what the bucketing kernels sort
    const uint4* rsorted;         // rrec grouped by node (stable; .y replaced by the running-pod index), node n's at list_off[n]
    const uint32_t* list_off;
    uint4* vlist;                 // each node's list by priority descending, then index: {claims, index, first claim, prio}
    const uint4* inv; const uint32_t* node_off; uint32_t n_node, n_gpu; const uint32_t* tbl; SelCtx sel;
    uint32_t exhaustive;
    uint4* psum;                  // [n_pair] {status | violations << PRE_VSHIFT, victims, highest victim priority, lowest
                                  //  running index among the victims of that priority}
    unsigned long long* psum64;   // [n_pair] sum over the victims of (priority + 2^31)
    uint8_t* pair_status; uint32_t* pair_victims;                   // caller's per-pair outputs (may be nullptr)
    uint32_t* pod_node; uint8_t* pod_status; uint32_t* n_victims; uint32_t* choice;
    uint32_t max_victims;
    unsigned long long* work;     // next unclaimed pair (zeroed by the host)
    const uint32_t* gate;         // non-zero: the running pods failed their check, nothing is evaluated
    Err err;
    // disruption budgets (spec §14, "Disruption budgets"; dra_preempt_pdb_batch), all nullptr / 0 without them
    const uint32_t* run_pdb;      // [rn_pod] each running pod's budget, or DRA_PDB_NONE (checked by k_pre_running)
    const int32_t* pdb_allowed;   // [n_pdb] disruptionsAllowed
    uint32_t n_pdb;
    uint32_t pdb;                 // non-zero: budgets in force (n_pdb > 0, running pods): vprev is built and read
    uint32_t* vprev;              // [rn_pod] per vlist position, the previous position of its node's list with the same budget
    uint32_t* pair_viol; uint32_t* pod_viol;                        // caller's violation outputs (may be nullptr)
};

// psum[k].x and the sharded call's pair records hold status | violations << PRE_VSHIFT (a status takes 3 bits; the
// violations fit the other 29 because a budgeted call has fewer than 2^29 running pods)
constexpr uint32_t PRE_VSHIFT = 3, PRE_ST_MASK = (1u << PRE_VSHIFT) - 1u;

// The pair kernel's node window and the sharded call's partials (layout at k_spre_reduce).  The single-inventory call:
// the window [0, n_node), n_walk = n_pair, no partials.
struct PreShard {
    uint32_t node_lo, n_win;      // the pairs to judge are those of the nodes in [node_lo, node_lo + n_win), or of no node
    uint32_t n_walk;              // pairs the evaluation walks: dense n_pod * n_win, else n_pair
    uint32_t stride;              // uint4 units per pod partial: 2 + ceil(max_victims / 4)
    uint4* part;                  // the partials (header, pods)
    uint2* pairs;                 // the window's pair results (nullptr: the caller asked for none)
};

// Thread per running pod.  Its node is the node of the GPUs its OK slots name (slots counted as §9 counts them); a pod
// without an OK slot is on no node.  Offsets not monotone or not spanning, a slot range outside rn_out, a GPU index
// >= n_gpu or GPUs of two nodes set ERR_BAD_OFFSETS, which gates every kernel after the sort; so does a budget that is
// neither DRA_PDB_NONE nor below n_pdb.
__global__ void __launch_bounds__(256)
k_pre_running(const PreArgs a) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0 && (__ldg(&a.rpod_off[0]) != 0 || __ldg(&a.rpod_off[a.rn_pod]) != a.rn_claim)) a.err.set(ERR_BAD_OFFSETS);
    if (r >= a.rn_pod) return;
    const uint32_t c0 = __ldg(&a.rpod_off[r]), c1 = __ldg(&a.rpod_off[r + 1]);
    const bool have_off = a.rout_off != nullptr;
    uint32_t node = DRA_GPU_NONE;
    bool bad = c1 < c0 || c1 > a.rn_claim;
    if (a.run_pdb) {
        const uint32_t b = __ldg(&a.run_pdb[r]);
        bad = bad || (b != DRA_PDB_NONE && b >= a.n_pdb);
    }
    for (uint32_t i = c0; !bad && i < c1; ++i) {
        const uint4 c = __ldg(&a.rclaims[i]);
        const uint32_t base = have_off ? __ldg(&a.rout_off[i]) : i, slots = dealloc_slots(c, a.n_node, have_off);
        if (base > a.rn_out || slots > a.rn_out - base) { bad = true; break; }
        for (uint32_t k = 0; k < slots; ++k) {
            const uint2 o = __ldg(&a.rout[base + k]);
            if ((o.y >> 24) != DRA_ST_OK) continue;
            if (o.x >= a.n_gpu) { bad = true; break; }
            const uint32_t n = __ldg(&a.inv[o.x]).z;
            if (node == DRA_GPU_NONE) node = n;
            else if (node != n) { bad = true; break; }
        }
    }
    if (bad) { a.err.set(ERR_BAD_OFFSETS); node = DRA_GPU_NONE; }
    a.rrec[r] = make_uint4(bad ? 0u : c1 - c0, node, c0, (uint32_t)__ldg(&a.rprio[r]));
}

// CTA per node: the node's running pods (index order after the stable bucketing) ranked by (priority descending, index
// ascending), a total order, so each pod's rank is the number of pods before it.  Quadratic in the pods of one node.
// With budgets, then each list position's previous position with the same budget (vprev; NONE for none or no budget),
// also quadratic at worst.
__global__ void __launch_bounds__(256)
k_pre_vsort(const PreArgs a) {
    if (__ldcg(a.gate)) return;
    for (uint32_t n = blockIdx.x; n < a.n_node; n += gridDim.x) {
        const uint32_t l0 = __ldcg(&a.list_off[n]), l1 = __ldcg(&a.list_off[n + 1]);
        for (uint32_t e = l0 + threadIdx.x; e < l1; e += blockDim.x) {
            const uint4 me = __ldcg(&a.rsorted[e]);
            uint32_t rank = 0;
            for (uint32_t f = l0; f < l1; ++f) {
                const uint4 o = __ldcg(&a.rsorted[f]);
                rank += ((int32_t)o.w > (int32_t)me.w || ((int32_t)o.w == (int32_t)me.w && o.y < me.y)) ? 1u : 0u;
            }
            a.vlist[l0 + rank] = me;
        }
        if (!a.pdb) continue;
        __syncthreads();                                                 // the node's list is in place
        for (uint32_t e = l0 + threadIdx.x; e < l1; e += blockDim.x) {
            const uint32_t b = __ldg(&a.run_pdb[__ldcg(&a.vlist[e]).y]);
            uint32_t prev = DRA_GPU_NONE;
            for (uint32_t f = e; b != DRA_PDB_NONE && f-- > l0;)
                if (__ldg(&a.run_pdb[__ldcg(&a.vlist[f]).y]) == b) { prev = f; break; }
            a.vprev[e] = prev;
        }
    }
}

// Running pod v = {claims, -, first claim, -} applied to this lane's GPU (global index gidx, NONE for a lane without one):
// add = the Allocate updates, else their §9 inverse, in the records' u16 / u32 arithmetic.
__device__ __forceinline__ void pre_apply(Lane& L, const PreArgs& a, const uint4 v, const uint32_t gidx, const bool add) {
    const bool have_off = a.rout_off != nullptr;
    for (uint32_t i = v.z; i < v.z + v.x; ++i) {
        const uint4 c = __ldg(&a.rclaims[i]);
        const uint32_t kind = c.x & 0xFFu;
        const uint32_t base = have_off ? __ldg(&a.rout_off[i]) : i, slots = dealloc_slots(c, a.n_node, have_off);
        for (uint32_t k = 0; k < slots; ++k) {
            const uint2 o = __ldg(&a.rout[base + k]);
            if ((o.y >> 24) != DRA_ST_OK || o.x != gidx) continue;
            if (kind == DRA_KIND_GPU) {
                L.flags = add ? (L.flags | DRA_GPU_FULL_ALLOCATED) : (L.flags & ~(uint32_t)DRA_GPU_FULL_ALLOCATED);
            } else if (kind == DRA_KIND_MIG) {
                const uint32_t m = slice_mask(o.y & 0xFFu, (o.y >> 8) & 0xFFu);
                L.busy = add ? (L.busy | m) : (L.busy & ~m);
            } else if (kind == DRA_KIND_SHARED) {
                L.mem = add ? L.mem - c.z : L.mem + c.z;
                L.share = (add ? L.share + 1u : L.share - 1u) & 0xFFFFu;
            }
        }
    }
}

// A pair's summary: status, victims, the highest victim priority and the lowest running index among the victims of that
// priority, the sum of (priority + 2^31) over the victims, and the victims whose eviction violates a budget
struct PreSum { uint32_t st, count, hi, hi_idx; unsigned long long sum; uint32_t viol; };

// Is V's member at list position v (running pod y) violating (spec §14, "Disruption budgets"): do the members in the list
// positions [v0, v] that count against its budget b number more than allowed[b]?  Walks b's chain back from v through
// vprev, at most allowed[b] steps.  The same on every lane.
__device__ __forceinline__ bool pre_violating(const PreArgs& a, const uint32_t v0, uint32_t v, const uint32_t y) {
    const uint32_t b = __ldg(&a.run_pdb[y]);
    if (b == DRA_PDB_NONE) return false;
    const int32_t allowed = __ldg(&a.pdb_allowed[b]);
    if (allowed < 0) return true;
    for (uint32_t n = 0; n < (uint32_t)allowed; ++n) {                   // n + 1 members of b found in [v, v1)
        v = __ldcg(&a.vprev[v]);
        if (v == DRA_GPU_NONE || v < v0) return false;
    }
    return true;
}

// Is the pod of cnt claims at `claims` INVALID: more than DRA_MAX_POD claims, or one invalid in slot mode have_off (§1) or
// naming a selector past n_sel?  On the W lanes gbase.. (gl = lane - gbase; gmask the group's lanes), answered on each.
template <int W>
__device__ __forceinline__ bool pod_invalid(const uint4* claims, const uint32_t cnt, const uint32_t n_sel, const bool have_off,
                                            const uint32_t gl, const uint32_t gmask) {
    bool inv = cnt > DRA_MAX_POD;
    for (uint32_t i = gl; i < cnt && !inv; i += W) {
        const uint4 c = __ldg(&claims[i]);
        const uint32_t kind = c.x & 0xFFu, prof = (c.x >> 8) & 0xFFu, count = c.x >> 16;
        inv = claim_invalid(kind, prof, count, have_off) || claim_sel(kind, c.z, c.w) > n_sel;
    }
    return (__ballot_sync(gmask, inv) & gmask) != 0u;
}

// Pair (pod, node) on the W lanes gbase.. of the warp.  skip_first: the pair is known to be EVICT (k_pods_preempt_victims), so the
// evaluation on the node as it is and the validity check are left out.  row: where the victims go (lane gbase writes).
// LIVE (spec §15, k_pods_preempt_place): the node as it stands is *live, the walk's working state, instead of a.inv; `row` is
// then the call's evicted-by word per running pod: running pods whose word is set are gone and left out of V, and with
// skip_first each victim's word is set to `pod`.  Lane gbase writes the words and its reading decides for the group.
template <int W, bool LIVE = false>
__device__ __forceinline__ PreSum pre_pair(const PreArgs& a, const uint32_t* __restrict__ tbl_s, const uint32_t pod,
                                           const uint32_t node, const uint32_t lane, const uint32_t gmask, const uint32_t gbase,
                                           const bool skip_first, uint32_t* row, const Lane* live = nullptr) {
    PreSum s{DRA_PRE_NO, 0u, 0x80000000u, 0xFFFFFFFFu, 0ull, 0u};
    if (node >= a.n_node) return s;
    const uint32_t c0 = __ldg(&a.pod_off[pod]), cnt = __ldg(&a.pod_off[pod + 1]) - c0;
    if (cnt > DRA_MAX_POD) { s.st = DRA_PRE_INVALID; return s; }
    const uint32_t gl = lane - gbase;
    const uint32_t g0 = __ldg(&a.node_off[node]), ng = __ldg(&a.node_off[node + 1]) - g0;
    if (ng > W) return s;                                             // cannot happen: W is chosen from the inventory
    const uint32_t gidx = gl < ng ? g0 + gl : DRA_GPU_NONE;
    Lane L;
    if constexpr (LIVE) L = *live;
    else L.load(gl < ng ? __ldg(&a.inv[g0 + gl]) : make_uint4(0, 0, 0, 0), gl < ng);
    const PodGet get{a.claims + c0, nullptr, 0};
    const bool exh = a.exhaustive != 0;
    uint32_t st1 = DRA_ST_POD;
    Lane Lt;                                                          // ONE copy handed to every pod_eval: one stack slot
    if (!skip_first) {
        Lt = L;
        st1 = pod_eval<W>(Lt, lane, gmask, gbase, g0, tbl_s, get, cnt, a.sel, exh, true, nullptr);
        if (st1 == 0) { s.st = DRA_PRE_FITS; return s; }
        if (pod_invalid<W>(a.claims + c0, cnt, a.sel.n_sel, true, gl, gmask)) { s.st = DRA_PRE_INVALID; return s; }
    }
    // V: the tail of the node's list below the pod's priority (the list is by priority descending)
    const int32_t P = __ldg(&a.prio[pod]);
    uint32_t v0 = __ldcg(&a.list_off[node]), hi = __ldcg(&a.list_off[node + 1]);
    const uint32_t v1 = hi;
    while (v0 < hi) {
        const uint32_t mid = (v0 + hi) >> 1;
        if ((int32_t)__ldcg(&a.vlist[mid]).w >= P) v0 = mid + 1; else hi = mid;
    }
    if (v0 == v1) { s.st = st1 == DRA_ST_SEARCH_LIMIT ? DRA_PRE_SEARCH_LIMIT : DRA_PRE_NO; return s; }   // S' = S
    bool any = !LIVE;
    for (uint32_t v = v0; v < v1; ++v) {
        const uint4 r = __ldcg(&a.vlist[v]);
        if constexpr (LIVE) { if (__shfl_sync(gmask, __ldcg(&row[r.y]), gbase) != DRA_GPU_NONE) continue; any = true; }
        pre_apply(L, a, r, gidx, false);
    }
    if (!any) { s.st = st1 == DRA_ST_SEARCH_LIMIT ? DRA_PRE_SEARCH_LIMIT : DRA_PRE_NO; return s; }   // every member gone: S' = S
    {
        Lt = L;
        const uint32_t st = pod_eval<W>(Lt, lane, gmask, gbase, g0, tbl_s, get, cnt, a.sel, exh, true, nullptr);
        if (st != 0) { s.st = st == DRA_ST_SEARCH_LIMIT ? DRA_PRE_SEARCH_LIMIT : DRA_PRE_NO; return s; }
    }
    s.st = DRA_PRE_EVICT;
    if constexpr (!LIVE) {
        if (a.pdb) {
            // Budgets: the reprieve over V's violating members first, then over the others, each phase in V order.
            // keep(S, r): r re-applied to S; true, with S updated, if the pod still fits there.
            auto keep = [&](Lane& S, const uint4 r) {
                Lane Lk = S;
                pre_apply(Lk, a, r, gidx, true);
                Lt = Lk;
                if (pod_eval<W>(Lt, lane, gmask, gbase, g0, tbl_s, get, cnt, a.sel, exh, true, nullptr) != 0) return false;
                S = Lk;
                return true;
            };
            auto victim = [&](const uint4 r, const bool vf) {           // victims come out of V order: true max / min
                if (s.count == 0 || (int32_t)r.w > (int32_t)s.hi || (r.w == s.hi && r.y < s.hi_idx)) { s.hi = r.w; s.hi_idx = r.y; }
                s.sum += (unsigned long long)((long long)(int32_t)r.w + 2147483648ll);
                if (row && s.count < a.max_victims && lane == gbase) row[s.count] = r.y;
                s.viol += vf ? 1u : 0u;
                ++s.count;
            };
            if (!row) {                                              // the counts: both phases on L
                for (uint32_t v = v0; v < v1; ++v) {
                    const uint4 r = __ldcg(&a.vlist[v]);
                    if (pre_violating(a, v0, v, r.y) && !keep(L, r)) victim(r, true);
                }
                for (uint32_t v = v0; v < v1; ++v) {
                    const uint4 r = __ldcg(&a.vlist[v]);
                    if (!pre_violating(a, v0, v, r.y) && !keep(L, r)) victim(r, false);
                }
            } else {
                // The victims in V order: the violating phase once for its end state Lb, then V once with two states,
                // L replaying the violating phase and Lb the other one, each member deciding on its own phase's state
                Lane Lb = L;
                for (uint32_t v = v0; v < v1; ++v) {
                    const uint4 r = __ldcg(&a.vlist[v]);
                    if (pre_violating(a, v0, v, r.y)) (void)keep(Lb, r);
                }
                for (uint32_t v = v0; v < v1; ++v) {
                    const uint4 r = __ldcg(&a.vlist[v]);
                    const bool vf = pre_violating(a, v0, v, r.y);
                    if (!(vf ? keep(L, r) : keep(Lb, r))) victim(r, vf);
                }
            }
            return s;
        }
    }
    for (uint32_t v = v0; v < v1; ++v) {                            // the reprieve, most important first
        const uint4 r = __ldcg(&a.vlist[v]);
        if constexpr (LIVE) { if (__shfl_sync(gmask, __ldcg(&row[r.y]), gbase) != DRA_GPU_NONE) continue; }
        Lane Lk = L;
        pre_apply(Lk, a, r, gidx, true);
        Lt = Lk;
        if (pod_eval<W>(Lt, lane, gmask, gbase, g0, tbl_s, get, cnt, a.sel, exh, true, nullptr) == 0) { L = Lk; continue; }
        if (s.count == 0) { s.hi = r.w; s.hi_idx = r.y; }            // V order: the first victim has the highest priority
        s.sum += (unsigned long long)((long long)(int32_t)r.w + 2147483648ll);
        if constexpr (LIVE) { if (skip_first && lane == gbase) row[r.y] = pod; }
        else { if (row && s.count < a.max_victims && lane == gbase) row[s.count] = r.y; }
        ++s.count;
    }
    return s;
}

// W lanes per (pod, candidate) pair, 32/W pairs per warp, in k_unsuitable's layout; pairs are taken from a counter, since
// a pair costs from one evaluation to |V| + 2 of them.  The pairs of s's node window (pair_decode); a pair naming no node
// is judged NO, as k_pre_choose reads every pair.
template <int WPC, int W>
__global__ void __launch_bounds__(WPC * 32, 2)
k_pods_preempt(const PreArgs a, const PreShard s) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    if (__ldcg(a.gate)) return;
    stage_table<WPC * 32>(tbl_s, a.tbl);
    constexpr uint32_t G = 32 / W;
    const auto [lane, grp, gl, gbase, gmask] = lane_group<W>();
    while (true) {
        const uint32_t pw = walk_fetch<G>(a.work, lane);
        if (pw >= s.n_walk) break;
        const uint32_t walk = pw + grp;
        if (walk >= s.n_walk) continue;                                  // whole group skips together
        uint32_t pod, node, pair;
        if (!pair_decode(walk, s.node_lo, s.n_win, a.n_node, a.cand_off, a.cand_nodes, a.pair_pod, pod, node, pair)) continue;
        const PreSum r = pre_pair<W>(a, tbl_s, pod, node, lane, gmask, gbase, false, nullptr);
        if (lane == gbase) {
            const uint32_t nv = r.st == DRA_PRE_EVICT ? r.count : 0u;   // (r.viol is 0 unless EVICT)
            a.psum[pair] = make_uint4(r.st | r.viol << PRE_VSHIFT, r.count, r.hi, r.hi_idx);
            a.psum64[pair] = r.sum;
            if (a.pair_status) a.pair_status[pair] = (uint8_t)r.st;
            if (a.pair_victims) a.pair_victims[pair] = nv;
            if (a.pair_viol) a.pair_viol[pair] = r.viol;
            if (s.pairs) s.pairs[pair] = make_uint2(r.st | r.viol << PRE_VSHIFT, nv);
        }
    }
}

// is EVICT pair x (summary xs, sum x64) preferred to y?  Equal summaries: neither (list position decides)
__device__ __forceinline__ bool pre_better(const uint4 xs, const unsigned long long x64, const uint4 ys, const unsigned long long y64) {
    if (xs.x >> PRE_VSHIFT != ys.x >> PRE_VSHIFT) return xs.x >> PRE_VSHIFT < ys.x >> PRE_VSHIFT;   // fewest violations
    if (xs.z != ys.z) return (int32_t)xs.z < (int32_t)ys.z;             // lowest highest victim priority
    if (x64 != y64) return x64 < y64;                                    // lowest sum of priorities
    if (xs.y != ys.y) return xs.y < ys.y;                                // fewest victims
    return xs.w > ys.w;                                                  // latest "start" among the highest-priority victims
}

// Warp-wide: every lane ends with the warp's preferred EVICT candidate (position best, NONE for none; summary bs, its
// .x the violations << PRE_VSHIFT with any status bits; sum b64), ties to the lower position.
__device__ __forceinline__ void pre_best_warp(uint32_t& best, uint4& bs, unsigned long long& b64) {
    for (uint32_t d = 16; d; d >>= 1) {
        const uint32_t ob = __shfl_xor_sync(FULLMASK, best, d);
        uint4 os;
        os.x = __shfl_xor_sync(FULLMASK, bs.x, d); os.y = __shfl_xor_sync(FULLMASK, bs.y, d);
        os.z = __shfl_xor_sync(FULLMASK, bs.z, d); os.w = __shfl_xor_sync(FULLMASK, bs.w, d);
        const unsigned long long o64 = __shfl_xor_sync(FULLMASK, b64, d);
        const bool take = ob != DRA_GPU_NONE &&
                          (best == DRA_GPU_NONE || pre_better(os, o64, bs, b64) || (!pre_better(bs, b64, os, o64) && ob < best));
        if (take) { best = ob; bs = os; b64 = o64; }
    }
}

struct PreScan { uint32_t fit, best; uint4 bs; unsigned long long b64; bool lim; };

// Warp-wide, the pair summaries psum[k0 .. k1) in list order (with win_nodes, only the pairs k whose node win_nodes[k] lies
// in [lo, lo + n_win)): the first FITS position, the preferred EVICT position with its summary and sum, and whether a
// SEARCH_LIMIT was seen.  The same on every lane.
__device__ __forceinline__ PreScan pre_scan(const PreArgs& a, const uint32_t k0, const uint32_t k1, const uint32_t lane,
                                            const uint32_t* win_nodes = nullptr, const uint32_t lo = 0, const uint32_t n_win = 0) {
    PreScan r{DRA_GPU_NONE, DRA_GPU_NONE, make_uint4(0, 0, 0, 0), 0ull, false};
    for (uint32_t j = k0 + lane; j < k1; j += 32) {                      // each lane in list order: ties keep the earlier
        if (win_nodes && __ldg(&win_nodes[j]) - lo >= n_win) continue;
        const uint4 s = __ldcg(&a.psum[j]);
        const uint32_t st = s.x & PRE_ST_MASK;
        if (st == DRA_PRE_FITS) r.fit = min(r.fit, j);
        else if (st == DRA_PRE_SEARCH_LIMIT) r.lim = true;
        else if (st == DRA_PRE_EVICT) {
            const unsigned long long v = __ldcg(&a.psum64[j]);
            if (r.best == DRA_GPU_NONE || pre_better(s, v, r.bs, r.b64)) { r.best = j; r.bs = s; r.b64 = v; }
        }
    }
    r.fit = __reduce_min_sync(FULLMASK, r.fit);
    r.lim = __any_sync(FULLMASK, r.lim);
    pre_best_warp(r.best, r.bs, r.b64);
    return r;
}

// The pod's status from its reduced pairs: FITS at the first such pair, else the preferred EVICT pair, else INVALID /
// SEARCH_LIMIT / NO.  k = the chosen position (NONE without one).
__device__ __forceinline__ uint32_t pre_decide(const uint32_t fit, const uint32_t best, const bool lim, const bool inv, uint32_t& k) {
    k = DRA_GPU_NONE;
    if (fit != DRA_GPU_NONE) { k = fit; return DRA_PRE_FITS; }
    if (best != DRA_GPU_NONE) { k = best; return DRA_PRE_EVICT; }
    return inv ? DRA_PRE_INVALID : lim ? DRA_PRE_SEARCH_LIMIT : DRA_PRE_NO;
}

// Warp-wide, pod p's pairs psum[k0 .. k1) reduced and decided.  Returns the status; k = the chosen pair, bs = its summary.
__device__ __forceinline__ uint32_t pre_reduce(const PreArgs& a, const uint32_t p, const uint32_t k0, const uint32_t k1,
                                               const uint32_t lane, uint32_t& k, uint4& bs) {
    const PreScan r = pre_scan(a, k0, k1, lane);
    const uint32_t c0 = __ldg(&a.pod_off[p]), cnt = __ldg(&a.pod_off[p + 1]) - c0;
    const bool inv = pod_invalid<32>(a.claims + c0, cnt, a.sel.n_sel, true, lane, FULLMASK);
    bs = r.bs;
    return pre_decide(r.fit, r.best, r.lim, inv, k);
}

// Warp per pod: its pairs reduced by pre_reduce.
__global__ void __launch_bounds__(256)
k_pre_choose(const PreArgs a) {
    if (__ldcg(a.gate)) return;
    const uint32_t lane = threadIdx.x & 31, p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p >= a.n_pod) return;
    uint32_t k0, k1;
    pod_pairs(a.cand_off, p, a.n_node, 0u, a.n_node, k0, k1);
    uint32_t k; uint4 bs;
    const uint32_t st = pre_reduce(a, p, k0, k1, lane, k, bs);
    if (lane != 0) return;
    a.pod_status[p] = (uint8_t)st;
    a.pod_node[p] = k == DRA_GPU_NONE ? DRA_GPU_NONE : pair_node(a.cand_off, a.cand_nodes, k, p, a.n_node);
    a.n_victims[p] = st == DRA_PRE_EVICT ? bs.y : 0u;
    if (a.pod_viol) a.pod_viol[p] = st == DRA_PRE_EVICT ? bs.x >> PRE_VSHIFT : 0u;
    a.choice[p] = st == DRA_PRE_EVICT ? k : DRA_GPU_NONE;
}

// W lanes per pod p whose chosen EVICT pair is choice[p * cstride] (NONE: none): its reprieve once more, writing the first
// min(count, max_victims) victims into the row at rows + p * rstride (the rest is filled by the caller).  Deterministic, so
// the victims are the ones k_pods_preempt counted.
template <int WPC, int W>
__global__ void __launch_bounds__(WPC * 32, 2)
k_pods_preempt_victims(const PreArgs a, const uint32_t* choice, const uint32_t cstride, uint32_t* rows, const uint32_t rstride) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    if (__ldcg(a.gate)) return;
    stage_table<WPC * 32>(tbl_s, a.tbl);
    constexpr uint32_t G = 32 / W;
    const uint32_t wid = threadIdx.x >> 5;
    const auto [lane, grp, gl, gbase, gmask] = lane_group<W>();
    for (uint32_t pw = (blockIdx.x * WPC + wid) * G; pw < a.n_pod; pw += gridDim.x * WPC * G) {
        const uint32_t p = pw + grp;
        if (p >= a.n_pod) continue;
        const uint32_t k = __ldcg(&choice[(size_t)p * cstride]);
        if (k == DRA_GPU_NONE) continue;
        const uint32_t node = pair_node(a.cand_off, a.cand_nodes, k, p, a.n_node);
        (void)pre_pair<W>(a, tbl_s, p, node, lane, gmask, gbase, true, rows + (size_t)p * rstride);
    }
}

// ---- preempt and place (spec §15, dra_preempt_place_batch) ---------------------------------------------------------
// §14's pair judgement and choice inside §13's walk: pods in input order, each judged on the nodes as the pods before it
// left them.  k_pre_running, the counting sort and k_pre_vsort build each node's running list as for §14; k_pp_prep and
// the counting sort build each node's visit list as for §13.  Then k_pods_preempt_place: a warp owns whole nodes, one lane
// per GPU, with a cursor into each node's visit list.  At pod q's entry the owner judges the pair on the node as it
// stands (pre_pair<32, true>: V without the running pods that earlier pods evicted), publishes the summary into q's psum
// slots and counts q's open pairs down; the warp that publishes the last one reduces them (pre_reduce, list order) and
// releases the decision into q's state word.  A node passes q only once q is decided.  The chosen node first applies q:
// the chosen pair's reprieve once more (deterministic: nothing changed the node since), which marks the victims, §9 for
// each of them, then the §12 evaluation with OutRecs.  q's entries on a node are consecutive after the stable sort and are
// judged once: nothing changes the node between them.
//   Exact: a node judges or applies q only after every earlier pod that lists the node is decided and, if it chose the
//   node, applied there; a pod changes no node but the one it chose.
//   Progress: every node that lists the lowest undecided pod can reach it (every entry before it belongs to a decided pod),
//   so with every CTA resident its last pair is always judged.
// State word: PP_OPEN undecided; PP_NOWHERE decided, applied nowhere; else the chosen position (the node in the dense form)
// | PP_EVICT for an EVICT choice.
constexpr uint32_t PP_OPEN = 0xFFFFFFFFu, PP_NOWHERE = 0x80000000u, PP_EVICT = 0x40000000u;

struct PpArgs {
    uint32_t* pending;            // [n_pod] the pod's pairs not judged yet
    uint32_t* evicted_by;         // [rn_pod] the pod that evicted the running pod, or NONE (the caller's output)
    uint32_t* judged;             // [n_node] 1 + the last pod judged at the node
};

// Warp per pod: state word, open-pair count, pair records (candidate form; pairs naming no node are NO and carry node
// NONE, so the sort drops them, as do every pair of a pod that is never judged).  A pod that is never judged is decided
// here: an empty pod is FITS on its first candidate naming a node, with nothing written; a pod of more than 32 claims, or
// with a claim invalid in the call's slot mode (a GPU claim of count != 1 without out_off), is INVALID; a pod with no
// candidate naming a node is NO.  (The pair judgement assumes out_off: it must never see a pod the apply would reject.)
__device__ __forceinline__ void pp_prep_pod(const PreArgs& a, const PlaceArgs& pl, const PpArgs& pp, uint32_t p, uint32_t lane) {
    const uint32_t c0 = __ldg(&pl.pod_off[p]), cnt = __ldg(&pl.pod_off[p + 1]) - c0;
    const bool inv = pod_invalid<32>(pl.claims + c0, cnt, a.sel.n_sel, pl.out_off != nullptr, lane, FULLMASK);
    const bool live = cnt != 0 && !inv;
    uint32_t first = DRA_GPU_NONE, usable = 0;
    if (!pl.cand_off) {
        usable = pl.n_node;
        if (pl.n_node) first = 0;
    } else {
        const uint32_t k0 = __ldg(&pl.cand_off[p]), nk = __ldg(&pl.cand_off[p + 1]) - k0;
        for (uint32_t j0 = 0; j0 < nk; j0 += 32) {
            const uint32_t j = j0 + lane;
            const uint32_t n = j < nk ? __ldg(&pl.cand_nodes[k0 + j]) : DRA_GPU_NONE;
            const bool ok = n < pl.n_node;
            if (j < nk) {
                pl.pairs[k0 + j] = make_uint4(p, live && ok ? n : DRA_GPU_NONE, j, 0);
                if (!ok) { a.psum[k0 + j] = make_uint4(DRA_PRE_NO, 0, 0x80000000u, DRA_GPU_NONE); a.psum64[k0 + j] = 0; }
            }
            const uint32_t b = __ballot_sync(FULLMASK, ok);
            usable += (uint32_t)__popc(b);
            if (b && first == DRA_GPU_NONE) first = __shfl_sync(FULLMASK, n, __ffs(b) - 1);
        }
    }
    const bool judged = live && usable != 0;
    if (lane == 0) {
        pp.pending[p] = usable;
        pl.state[p] = judged ? PP_OPEN : PP_NOWHERE;
        if (!judged) {
            a.pod_node[p] = cnt == 0 ? first : DRA_GPU_NONE;
            a.pod_status[p] = (uint8_t)(cnt == 0 ? (first != DRA_GPU_NONE ? DRA_PRE_FITS : DRA_PRE_NO)
                                                 : inv ? DRA_PRE_INVALID : DRA_PRE_NO);
        }
    }
    if (cnt != 0 && !judged) place_fail(pl, c0, cnt, DRA_ST_POD, lane);
}

__global__ void __launch_bounds__(256)
k_pp_prep(const PreArgs a, const PlaceArgs pl, const PpArgs pp) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p >= pl.n_pod) return;
    pp_prep_pod(a, pl, pp, p, lane);
}

// Persistent: every CTA resident (cooperative launch); warp w owns nodes w, w + warps, ... and cycles over them.  Minimum
// one CTA per SM in the bounds: the walk's state beside pre_pair's then fits in registers without spilling (the stack
// holds only the two Lane copies handed to pod_eval).
template <int WPC>
__global__ void __launch_bounds__(WPC * 32, 1)
k_pods_preempt_place(const PreArgs a, const PlaceArgs pl, const PpArgs pp) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    if (__ldcg(a.gate)) return;
    stage_table<WPC * 32>(tbl_s, pl.tbl);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t w0 = blockIdx.x * WPC + (threadIdx.x >> 5), n_warp = gridDim.x * WPC;
    const bool dense = pl.cand_off == nullptr, have_off = pl.out_off != nullptr;
    uint32_t seen = 0;
    long long t0 = clock64();
    while (true) {
        bool left = false, moved = false;
        for (uint32_t node = w0; node < pl.n_node; node += n_warp) {
            const uint32_t l0 = dense ? 0u : __ldcg(&pl.list_off[node]), l1 = dense ? pl.n_pod : __ldcg(&pl.list_off[node + 1]);
            const uint32_t cur0 = l0 + __ldcg(&pl.cursor[node]);
            uint32_t cur = cur0;
            if (cur >= l1) continue;
            const uint32_t g0 = __ldg(&pl.node_off[node]), ng = __ldg(&pl.node_off[node + 1]) - g0;
            Lane L;
            bool loaded = false, dirty = false;
            while (cur < l1) {
                // 32 entries at once: the first one that is not to be skipped (decided, and not for this entry)
                const uint32_t e = cur + lane;
                uint32_t q = 0, k = 0, s = PP_NOWHERE;
                if (e < l1) {
                    if (dense) { q = e; k = node; }
                    else { const uint4 r = __ldcg(&pl.sorted[e]); q = r.x; k = r.z; }
                    s = ld_acquire_u32(&pl.state[q]);
                }
                const bool skip = s != PP_OPEN && ((s & PP_NOWHERE) || (s & PL_POS) != k);
                const uint32_t act = __ballot_sync(FULLMASK, !skip);
                if (!act) { cur = min(cur + 32u, l1); continue; }
                const uint32_t f = (uint32_t)__ffs(act) - 1u;
                cur += f;
                const uint32_t qf = __shfl_sync(FULLMASK, q, f), sf = __shfl_sync(FULLMASK, s, f);
                if (!loaded) {
                    L.load(lane < ng ? pl.inv_dst[g0 + lane] : make_uint4(0, 0, 0, 0), lane < ng);
                    loaded = true;
                }
                if (sf == PP_OPEN) {
                    if (__shfl_sync(FULLMASK, __ldcg(&pp.judged[node]), 0) == qf + 1u) break;   // judged, undecided: wait
                    // judge q here once, for each of its consecutive entries
                    const PreSum r = pre_pair<32, true>(a, tbl_s, qf, node, lane, FULLMASK, 0u, false, pp.evicted_by, &L);
                    const uint32_t kb = dense ? qf * pl.n_node : __ldg(&pl.cand_off[qf]);
                    uint32_t n_here = 0;
                    for (uint32_t e2 = cur; e2 < l1; ++e2) {
                        uint32_t pos = node;
                        if (!dense) { const uint4 r2 = __ldcg(&pl.sorted[e2]); if (r2.x != qf) break; pos = r2.z; }
                        else if (e2 != cur) break;
                        if (lane == 0) { a.psum[kb + pos] = make_uint4(r.st, r.count, r.hi, r.hi_idx); a.psum64[kb + pos] = r.sum; }
                        ++n_here;
                    }
                    __threadfence();
                    __syncwarp();
                    uint32_t last = 0;
                    if (lane == 0) {
                        pp.judged[node] = qf + 1u;
                        last = atomicSub(&pp.pending[qf], n_here) == n_here ? 1u : 0u;
                        atomicAdd(&pl.cursor[pl.n_node], 1u);
                    }
                    if (__shfl_sync(FULLMASK, last, 0)) {
                        // every pair of q is judged: the decision
                        __threadfence();
                        const uint32_t k0 = dense ? qf * pl.n_node : __ldg(&pl.cand_off[qf]);
                        const uint32_t k1 = dense ? k0 + pl.n_node : __ldg(&pl.cand_off[qf + 1]);
                        uint32_t kc; uint4 bs;
                        const uint32_t st = pre_reduce(a, qf, k0, k1, lane, kc, bs);
                        if (lane == 0) {
                            a.pod_status[qf] = (uint8_t)st;
                            a.pod_node[qf] = kc == DRA_GPU_NONE ? DRA_GPU_NONE : dense ? kc - k0 : __ldg(&pl.cand_nodes[kc]);
                        }
                        if (kc == DRA_GPU_NONE) {
                            const uint32_t c0 = __ldg(&pl.pod_off[qf]), cnt = __ldg(&pl.pod_off[qf + 1]) - c0;
                            place_fail(pl, c0, cnt, st == DRA_PRE_SEARCH_LIMIT ? (uint32_t)DRA_ST_SEARCH_LIMIT : (uint32_t)DRA_ST_POD, lane);
                        }
                        __threadfence();
                        __syncwarp();
                        if (lane == 0)
                            st_release_u32(&pl.state[qf], kc == DRA_GPU_NONE ? PP_NOWHERE : (kc - k0) | (st == DRA_PRE_EVICT ? PP_EVICT : 0u));
                    }
                    moved = true;
                    continue;                                        // q's state again: decided now, or this node waits
                }
                // q is decided, for this entry of this node: apply it
                const uint32_t c0 = __ldg(&pl.pod_off[qf]), cnt = __ldg(&pl.pod_off[qf + 1]) - c0;
                if (sf & PP_EVICT) {
                    (void)pre_pair<32, true>(a, tbl_s, qf, node, lane, FULLMASK, 0u, true, pp.evicted_by, &L);   // marks the victims
                    __syncwarp();
                    const uint32_t gidx = lane < ng ? g0 + lane : DRA_GPU_NONE;
                    const uint32_t v0 = __ldcg(&a.list_off[node]), v1 = __ldcg(&a.list_off[node + 1]);
                    for (uint32_t v = v0; v < v1; ++v) {             // §9 for each victim
                        const uint4 r = __ldcg(&a.vlist[v]);
                        if (__shfl_sync(FULLMASK, __ldcg(&pp.evicted_by[r.y]), 0) == qf) pre_apply(L, a, r, gidx, false);
                    }
                }
                {
                    const PodGet get{pl.claims + c0, have_off ? pl.out_off + c0 : nullptr, c0};
                    Lane Lt = L;
                    if (pod_eval<32>(Lt, lane, FULLMASK, 0, g0, tbl_s, get, cnt, pl.sel, pl.exhaustive != 0, have_off, pl.out) == 0) L = Lt;
                }
                dirty = true;
                __threadfence();
                __syncwarp();
                if (lane == 0) atomicAdd(&pl.cursor[pl.n_node], 1u);
                moved = true;
                ++cur;
            }
            if (dirty && lane < ng) pl.inv_dst[g0 + lane] = L.store(pl.inv_dst[g0 + lane]);    // (only this warp writes the node)
            if (cur != cur0) { moved = true; pl.cursor[node] = cur - l0; }
            if (cur < l1) left = true;
        }
        if (!left) break;
        if (moved) { t0 = clock64(); continue; }
        // nothing moved on this warp's nodes: back off, and give up when nothing moved anywhere for a long time (cannot
        // happen with every CTA resident)
        __nanosleep(256);
        const uint32_t pr = __shfl_sync(FULLMASK, ld_acquire_u32(&pl.cursor[pl.n_node]), 0);
        if (pr != seen) { seen = pr; t0 = clock64(); }
        else if (clock64() - t0 > 4000000000ll) {
            if (lane == 0) pl.err.set(ERR_DEVICE_WAIT);
            break;
        }
    }
}

// ---- preempt and place on a sharded world (dra_preempt_place_batch_global_device) -----------------------------------
// Every rank gets the same pending pods, candidates and running pods.  Each rank assembles the world's state in a scratch
// copy of the inventory: its own GPU range from its live copy, every other range from the owning rank over the inventory
// sync's exchange (k_peer_push of the live own range, k_isync_copy into the scratch copy).  Then every rank runs §15's
// chain on the scratch copy — k_pre_running, the counting sort, k_pre_vsort, k_spp_prep, the counting sort of the pairs and
// k_pods_preempt_place — so every rank takes the same decisions in the same order, and k_spp_final hands the caller the
// outputs and copies the rank's own GPU range back into its live copy.  The walk waits for no peer: the only wait is the
// exchange, before anything is judged.
struct SppArgs {
    uint32_t n_claim, n_pair, n_out;             // the pending arrays' lengths (n_pair 0: dense form)
    uint32_t* gate;                              // non-zero: a pending or running fault, or a peer missing; nothing is written
    const uint32_t* err_dev;                     // the context's device error words
    const uint32_t* pod_node_src; const uint8_t* pod_status_src; const uint32_t* evicted_src;   // the walk's outputs
    uint32_t* pod_node; uint8_t* pod_status; uint32_t* evicted_by;                          // the caller's
    uint32_t n_pod, rn_pod;
    const uint4* inv_src; uint4* inv_dst; uint32_t gpu_lo, gpu_hi;   // scratch -> live over this rank's GPU range
};

// One warp, after k_isync_copy: the world agrees on the exchange's verdict, so that the call fails on every rank or on
// none.  Lane p publishes this rank's verdict (its copy kernel's, `elect`[1], and no timeout here) to peer p as the flag
// {seq : ok}, then waits for peer p's.  A peer's failure, or a peer whose verdict does not arrive within the spin limit,
// closes the gate and sets ERR_PEER_TIMEOUT.  A rank that timed out in the exchange publishes its failure at once, before
// any peer that received everything can stop waiting for it here, so a late peer fails the call everywhere.
__global__ void __launch_bounds__(32)
k_spp_agree(const PeerExchange x, const uint32_t* __restrict__ elect, uint32_t sync_seq, uint32_t* gate) {
    const uint32_t tid = threadIdx.x;
    uint32_t v1;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v1) : "l"(elect + 1) : "memory");
    const uint32_t ok = (v1 == (sync_seq << 1 | 1u) && !__ldcg(&x.err.dev[ERR_PEER_TIMEOUT])) ? 1u : 0u;
    const uint32_t mine = x.seq << 1 | ok;
    bool fail = ok == 0u;
    if (tid < x.world && tid != x.rank) {
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(x.flag[tid]), "r"(mine) : "memory");
        const long long t0 = clock64();
        uint32_t v;
        while (true) {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(x.my_flags + tid) : "memory");
            if ((int32_t)((v >> 1) - x.seq) >= 0) { fail = fail || (v >> 1) != x.seq || !(v & 1u); break; }
            if (clock64() - t0 > x.spin_limit) { fail = true; break; }
        }
    }
    if (__any_sync(FULLMASK, fail) && tid == 0) { *gate = 1u; x.err.set(ERR_PEER_TIMEOUT); }
}

// Warp per pod: k_splace_prep's device-side checks of the pending arrays (pod_off and cand_off monotone and spanning them,
// at most PL_POS candidates, every claim's slots inside n_out, counted as dra_preempt_place_batch counts them), then
// k_pp_prep's work for a pod that passes.  A faulty pod sets ERR_BAD_OFFSETS and the gate and writes nothing.  Warp 0 also
// closes the gate on the faults found before it: the running pods' (k_pre_running) and a peer missing from the exchange.
__global__ void __launch_bounds__(256)
k_spp_prep(const PreArgs a, const PlaceArgs pl, const PpArgs pp, const SppArgs s) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p == 0 && lane == 0 && (__ldcg(&s.err_dev[ERR_BAD_OFFSETS]) || __ldcg(&s.err_dev[ERR_PEER_TIMEOUT]))) *s.gate = 1u;
    if (p >= pl.n_pod) return;
    const bool have_off = pl.out_off != nullptr;
    const uint32_t c0 = __ldg(&pl.pod_off[p]), c1 = __ldg(&pl.pod_off[p + 1]);
    bool fault = c1 < c0 || c1 > s.n_claim || (p == 0 && (c0 != 0 || __ldg(&pl.pod_off[pl.n_pod]) != s.n_claim));
    if (pl.cand_off) {
        const uint32_t k0 = __ldg(&pl.cand_off[p]), k1 = __ldg(&pl.cand_off[p + 1]);
        fault = fault || k1 < k0 || k1 > s.n_pair || k1 - k0 > PL_POS || (p == 0 && (k0 != 0 || __ldg(&pl.cand_off[pl.n_pod]) != s.n_pair));
    }
    if (!fault)
        for (uint32_t i = c0 + lane; i < c1; i += 32) {
            const uint4 c = __ldg(&pl.claims[i]);
            const uint32_t kind = c.x & 0xFFu, count = c.x >> 16;
            const bool gpu = kind == DRA_KIND_GPU && count >= 1 && count <= DRA_MAX_COUNT && (have_off || count == 1);
            const uint32_t slots = gpu ? count : 1u, dst = have_off ? __ldg(&pl.out_off[i]) : i;
            fault = fault || dst > s.n_out || slots > s.n_out - dst;
        }
    if (__any_sync(FULLMASK, fault)) {
        if (lane == 0) { *s.gate = 1u; a.err.set(ERR_BAD_OFFSETS); }
        return;
    }
    pp_prep_pod(a, pl, pp, p, lane);
}

// Grid-stride, after the walk: with the gate open and the walk complete, the caller's pod_node, pod_status and evicted_by
// from the walk's, and this rank's own GPU range from the scratch copy into the live one.  Otherwise nothing.
__global__ void __launch_bounds__(256)
k_spp_final(const SppArgs s) {
    if (__ldcg(s.gate) || __ldcg(&s.err_dev[ERR_DEVICE_WAIT])) return;
    const uint32_t t0 = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (uint32_t i = t0; i < s.n_pod; i += nt) { s.pod_node[i] = __ldcg(&s.pod_node_src[i]); s.pod_status[i] = __ldcg(&s.pod_status_src[i]); }
    for (uint32_t i = t0; i < s.rn_pod; i += nt) s.evicted_by[i] = __ldcg(&s.evicted_src[i]);
    for (uint32_t i = s.gpu_lo + t0; i < s.gpu_hi; i += nt) s.inv_dst[i] = __ldcg(&s.inv_src[i]);
}

// ---- sharded preemption (dra_preempt_batch_global_device) ----------------------------------------------------------
// Every rank gets the same pending pods, candidates and running pods.  k_uns_prep checks pod_off / cand_off and writes
// pair -> pod; k_pre_running, the counting sort and k_pre_vsort run unchanged on the whole inventory (their checks are
// on global GPU indices, so every rank finds the same fault).  Then, on this rank's node window only:
//   k_pods_preempt  the pair evaluation for the pairs whose node lies in the window (PreShard)
//   k_spre_reduce   warp per pod: k_pre_choose's reduction over the window's pairs, keeping list positions, into this
//                   rank's partial of the pod (and the rank's fault word into the partials' header)
//   k_pods_preempt_victims  W lanes per pod whose partial holds an EVICT pair and no FITS pair: that pair's victim row,
//                   the first min(count, max_victims) words (the merge fills the rest)
//   k_peer_push     the partials (and, when the caller asked for them, the window's pair results) to every peer
//   k_spre_merge    flags, wait, then per pod the minimum over the ranks' partials; writes the caller's buffers only if
//                   no rank reported a fault
// The partials, in uint4 units: [0] header {fault word}; pod p at 1 + p * stride: {fit position, best EVICT position,
// its victim count, its highest victim priority}, {its lowest victim index of that priority, SEARCH_LIMIT seen | its
// violations << 1, its priority sum lo, hi}, then the best pair's row of max_victims words; after the pods the window's
// pairs as {status | violations << PRE_VSHIFT, victims} (uint2).
// A position is the pair's index in the call's pair list, so the merge's choice is the minimum over the ranks of a total
// order — (FITS first, then pre_better, then position) — which is the single-inventory choice for any partition.
// k_pods_preempt also judges a candidate naming no node (NO); the reduce leaves it out and the merge writes it itself.
__global__ void __launch_bounds__(256)
k_spre_reduce(const PreArgs a, const PreShard s) {
    const uint32_t gate = __ldcg(a.gate);
    if (blockIdx.x == 0 && threadIdx.x == 0) s.part[0] = make_uint4(gate, 0u, 0u, 0u);
    if (gate) return;
    const uint32_t lane = threadIdx.x & 31, p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (p >= a.n_pod) return;
    uint32_t k0, k1;
    pod_pairs(a.cand_off, p, a.n_node, s.node_lo, s.n_win, k0, k1);
    PreScan r = pre_scan(a, k0, k1, lane, a.cand_off ? a.cand_nodes : nullptr, s.node_lo, s.n_win);
    if (lane != 0) return;
    if (r.fit != DRA_GPU_NONE) r.best = DRA_GPU_NONE;                    // a FITS pair anywhere beats every EVICT pair
    uint4* q = s.part + 1 + (size_t)p * s.stride;
    q[0] = make_uint4(r.fit, r.best, r.bs.y, r.bs.z);
    q[1] = make_uint4(r.bs.w, (r.lim ? 1u : 0u) | (r.bs.x >> PRE_VSHIFT) << 1, (uint32_t)r.b64, (uint32_t)(r.b64 >> 32));
}

struct PreMerge {
    const uint4* part;            // this rank's partials (PreShard::part); a peer's are at my_stage + sender * slice4
    const uint2* pairs;           // this rank's pair results; a peer's follow its partials in its slice
    uint32_t slice4, stride;      // uint4 units of one sender's slice; of one pod's partial
    const uint4* claims; const uint32_t* pod_off; uint32_t n_pod;
    const uint32_t* cand_nodes; const uint32_t* cand_off; uint32_t n_pair, n_node;
    SelCtx sel;
    uint32_t max_victims;
    uint32_t bounds[PEER_MAX + 1];   // rank r owns nodes [bounds[r], bounds[r + 1])
    const uint32_t* gate;            // this rank's fault word
    uint8_t* pair_status; uint32_t* pair_victims;                  // the caller's (pair outputs: nullptr unless asked)
    uint32_t* pod_node; uint8_t* pod_status; uint32_t* n_victims; uint32_t* victims;
    uint32_t* pair_viol; uint32_t* pod_viol;                        // the caller's violation outputs (nullptr: none)
};

// The start of a merge that waits for its peers (k_spre_merge, k_scap_merge): block 0 raises this rank's flags, every
// block waits, then every rank's fault word is read (this rank's at gate, a peer's in the first word of its slice, slice4
// uint4 units apart in x's staging).  A peer's fault fails the call here too.  False in every thread after a fault or a
// timeout: the merge writes nothing then.  world (at least 1), rank and tid as the kernel has them.
__device__ __forceinline__ bool merge_start(const PeerExchange& x, const uint32_t* gate, uint32_t slice4, uint32_t world,
                                            uint32_t rank, uint32_t tid) {
    __shared__ uint32_t s_ok;
    if (tid == 0) s_ok = 1u;
    __syncthreads();
    if (blockIdx.x == 0) peer_raise(x, tid);
    if (!peer_wait(x, tid, clock64())) s_ok = 0u;
    if (tid < world) {
        const uint32_t f = tid == rank ? __ldcg(gate) : __ldcg(&x.my_stage[(size_t)tid * slice4]).x;
        if (f) {
            s_ok = 0u;
            if (blockIdx.x == 0 && tid != rank) x.err.set(ERR_BAD_OFFSETS);
        }
    }
    __syncthreads();
    return s_ok != 0u;
}

// The rank whose node range [bounds[r], bounds[r + 1]) of the shard map holds node, in a world of world ranks
__device__ __forceinline__ uint32_t node_owner(const uint32_t* bounds, uint32_t world, uint32_t node) {
    uint32_t r = 0;
    while (r + 1 < world && bounds[r + 1] <= node) ++r;
    return r;
}

// At most SMs / 4 CTAs, launched after the evaluation: ranks sharing one device must not find their evaluation's SMs
// held by a peer's waiting CTAs.  Block 0 raises this rank's flags, every block waits; then a warp per pod (lane s reads
// rank s's partial) and a thread per pair.  With world 1 (an all-zero PeerExchange) nothing is waited for.
__global__ void __launch_bounds__(256)
k_spre_merge(const PeerExchange x, const PreMerge m) {
    const uint32_t tid = threadIdx.x, world = x.world ? x.world : 1u, rank = x.rank;
    if (!merge_start(x, m.gate, m.slice4, world, rank, tid)) return;
    const uint32_t lane = tid & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + tid) >> 5, n_warp = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t p = warp; p < m.n_pod; p += n_warp) {
        const uint4* src = nullptr;
        uint4 A = make_uint4(DRA_GPU_NONE, DRA_GPU_NONE, 0u, 0u), B = make_uint4(0u, 0u, 0u, 0u);
        if (lane < world) {
            src = (lane == rank ? m.part : x.my_stage + (size_t)lane * m.slice4) + 1 + (size_t)p * m.stride;
            A = __ldcg(&src[0]); B = __ldcg(&src[1]);
        }
        const uint32_t fit = __reduce_min_sync(FULLMASK, A.x);
        const bool lim = __any_sync(FULLMASK, (B.y & 1u) != 0u);
        uint32_t best = A.y;
        uint4 bs = make_uint4((B.y >> 1) << PRE_VSHIFT, A.z, A.w, B.x);
        unsigned long long b64 = (unsigned long long)B.z | ((unsigned long long)B.w << 32);
        pre_best_warp(best, bs, b64);
        const uint32_t c0 = __ldg(&m.pod_off[p]), cnt = __ldg(&m.pod_off[p + 1]) - c0;
        const bool inv = pod_invalid<32>(m.claims + c0, cnt, m.sel.n_sel, true, lane, FULLMASK);
        uint32_t k;
        const uint32_t st = pre_decide(fit, best, lim, inv, k);
        const uint32_t nv = st == DRA_PRE_EVICT ? bs.y : 0u;
        const uint32_t node = k == DRA_GPU_NONE ? DRA_GPU_NONE : pair_node(m.cand_off, m.cand_nodes, k, p, m.n_node);
        if (lane == 0) {
            m.pod_status[p] = (uint8_t)st;
            m.pod_node[p] = node;
            m.n_victims[p] = nv;
            if (m.pod_viol) m.pod_viol[p] = st == DRA_PRE_EVICT ? bs.x >> PRE_VSHIFT : 0u;
        }
        if (m.max_victims) {
            // the chosen EVICT pair's partial is its node's owner's (no row is read for any other status)
            const uint32_t win = st == DRA_PRE_EVICT ? node_owner(m.bounds, world, node) : rank;
            const uint32_t* row = reinterpret_cast<const uint32_t*>(
                (win == rank ? m.part : x.my_stage + (size_t)win * m.slice4) + 1 + (size_t)p * m.stride + 2);
            const uint32_t n = min(nv, m.max_victims);
            for (uint32_t j = lane; j < m.max_victims; j += 32)
                m.victims[(size_t)p * m.max_victims + j] = j < n ? __ldcg(&row[j]) : DRA_GPU_NONE;
        }
    }
    if (!m.pair_status && !m.pair_victims && !m.pair_viol) return;
    const size_t pair4 = 1 + (size_t)m.n_pod * m.stride;                 // a slice's pair results follow its partials
    for (uint32_t k = blockIdx.x * blockDim.x + tid; k < m.n_pair; k += gridDim.x * blockDim.x) {
        const uint32_t node = m.cand_off ? __ldg(&m.cand_nodes[k]) : k % m.n_node;
        uint2 v = make_uint2(DRA_PRE_NO, 0u);                             // a candidate naming no node
        if (node < m.n_node) {
            const uint32_t r = node_owner(m.bounds, world, node);
            const uint2* src = r == rank ? m.pairs : reinterpret_cast<const uint2*>(x.my_stage + (size_t)r * m.slice4 + pair4);
            v = __ldcg(&src[k]);
        }
        if (m.pair_status) m.pair_status[k] = (uint8_t)(v.x & PRE_ST_MASK);
        if (m.pair_victims) m.pair_victims[k] = v.y;
        if (m.pair_viol) m.pair_viol[k] = v.x >> PRE_VSHIFT;
    }
}

// ====================================================================================================
// Pod capacity (spec §16): how many copies of a pod each candidate node still takes
//   k_pods_capacity      W lanes per (pod, node) pair: pod_eval on a register copy of the node, the placement kept each
//                        time it succeeds, until one fails or max_copies are placed
//   k_pods_capacity_sum  warp per pod: the pod's pairs summed, and those with a copy counted
// The sharded call (dra_pod_capacity_batch_global_device) runs k_pods_capacity on its node window and k_scap_merge below.
// ====================================================================================================
struct CapArgs {
    const uint4* claims; const uint32_t* pod_off; uint32_t n_pod;
    const uint32_t* cand_nodes; const uint32_t* cand_off; const uint32_t* pair_pod;   // cand_off == nullptr: dense form
    uint32_t n_pair;
    const uint4* inv; const uint32_t* node_off; uint32_t n_node; const uint32_t* tbl; SelCtx sel;
    uint32_t exhaustive, max_copies;
    uint32_t node_lo, n_win, n_walk;   // the node window and the pairs walked, as in UnsArgs (one inventory: [0, n_node))
    uint16_t* pair_copies; uint8_t* pair_stop;            // at the walk index; pair_stop: nullptr unless asked for
    unsigned long long* pod_total; uint32_t* pod_nodes;   // each nullptr unless asked for
    unsigned long long* work;                             // next unclaimed pair (zeroed by the host)
    const uint32_t* gate;                                 // non-zero: the offsets failed their check (nullptr: none)
};

// k_pods_preempt's layout: W lanes per pair, 32/W pairs per warp, pairs taken from a counter, since a pair costs from one
// evaluation to max_copies of them.  One writer per pair, so the results are plain stores and nothing is zeroed first.
// A candidate naming no node, an empty pod and a pod of more than DRA_MAX_POD claims are answered without loading a node.
// The results go to the walk index (pair_decode's), which with the window [0, n_node) is the pair index in both forms.
template <int WPC, int W>
__global__ void __launch_bounds__(WPC * 32, 2)
k_pods_capacity(const CapArgs a) {
    __shared__ uint32_t tbl_s[DRA_MAX_MODELS * DRA_MAX_PROFILES];
    if (a.gate && __ldcg(a.gate)) return;
    stage_table<WPC * 32>(tbl_s, a.tbl);
    constexpr uint32_t G = 32 / W;
    const auto [lane, grp, gl, gbase, gmask] = lane_group<W>();
    while (true) {
        const uint32_t pw = walk_fetch<G>(a.work, lane);
        if (pw >= a.n_walk) break;
        const uint32_t walk = pw + grp;                                  // (results go to the walk index)
        if (walk >= a.n_walk) continue;                                  // whole group skips together
        // pair_decode's rule written out: through it, 76 registers instead of 74 and 11% slower at two ranks per device
        uint32_t pod, node;
        if (!a.cand_off) { pod = walk / a.n_win; node = a.node_lo + (walk - pod * a.n_win); }
        else {
            node = __ldg(&a.cand_nodes[walk]);
            if (node < a.n_node && node - a.node_lo >= a.n_win) continue;   // another rank's node
            pod = __ldg(&a.pair_pod[walk]);
        }
        const uint32_t c0 = __ldg(&a.pod_off[pod]), cnt = __ldg(&a.pod_off[pod + 1]) - c0;
        uint32_t copies = 0, stop = DRA_ST_POD;                           // a candidate naming no node: unsuitable (§8)
        if (node >= a.n_node) {}
        else if (cnt == 0) { copies = a.max_copies; stop = DRA_ST_OK; }
        else if (cnt > DRA_MAX_POD) stop = DRA_ST_INVALID;
        else {
            const uint32_t g0 = __ldg(&a.node_off[node]), ng = __ldg(&a.node_off[node + 1]) - g0;
            if (ng <= W) {                                                // always: W is chosen from the inventory
                Lane L; L.load(gl < ng ? __ldg(&a.inv[g0 + gl]) : make_uint4(0, 0, 0, 0), gl < ng);
                const PodGet get{a.claims + c0, nullptr, 0};
                Lane Lt;                                                  // ONE copy handed to every pod_eval: one stack slot
                stop = DRA_ST_OK;
                while (copies < a.max_copies) {
                    Lt = L;
                    const uint32_t st = pod_eval<W>(Lt, lane, gmask, gbase, g0, tbl_s, get, cnt, a.sel, a.exhaustive != 0, true, nullptr);
                    if (st) { stop = st; break; }
                    L = Lt; ++copies;
                }
                // validity does not depend on the node's state: an invalid pod fails its first evaluation
                if (stop == DRA_ST_POD && copies == 0 && pod_invalid<W>(a.claims + c0, cnt, a.sel.n_sel, true, gl, gmask))
                    stop = DRA_ST_INVALID;
            }
        }
        if (lane == gbase) {
            a.pair_copies[walk] = (uint16_t)copies;
            if (a.pair_stop) a.pair_stop[walk] = (uint8_t)stop;
        }
    }
}

// A warp's sums over pod p's pairs [k0, k1), the lanes striding them: copies(k) gives pair k's count.  The counts are 16
// bits each, so a lane's sum needs 64 bits only beyond 65,537 pairs per lane; it is kept in 64 bits throughout and reduced
// with a shuffle tree.
template <class F>
__device__ __forceinline__ void cap_pod_sums(uint32_t p, uint32_t lane, unsigned long long k0, unsigned long long k1, F copies,
                                             unsigned long long* pod_total, uint32_t* pod_nodes) {
    unsigned long long sum = 0;
    uint32_t nodes = 0;
    for (unsigned long long k = k0; k < k1; k += 32) {
        const uint32_t c = k + lane < k1 ? copies(k + lane) : 0u;
        sum += c;
        nodes += __popc(__ballot_sync(FULLMASK, c != 0u));
    }
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(FULLMASK, sum, d);
    if (lane == 0) {
        if (pod_total) pod_total[p] = sum;
        if (pod_nodes) pod_nodes[p] = nodes;
    }
}

// Warp per pod: the lanes stride the pod's pairs (dense: its row of n_node).
__global__ void __launch_bounds__(256)
k_pods_capacity_sum(const CapArgs a) {
    const uint32_t lane = threadIdx.x & 31, p = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (p >= a.n_pod) return;
    unsigned long long k0, k1;
    pod_pairs(a.cand_off, p, a.n_node, 0u, a.n_node, k0, k1);
    cap_pod_sums(p, lane, k0, k1, [&](unsigned long long k) { return (uint32_t)a.pair_copies[k]; }, a.pod_total, a.pod_nodes);
}

// ---- sharded pod capacity (dra_pod_capacity_batch_global_device) --------------------------------------------------
// Every rank gets the same pods and candidates.  k_uns_prep checks pod_off / cand_off and writes pair -> pod; its fault
// word gates k_pods_capacity, which evaluates this rank's window into its slice; k_peer_push sends the slice to every
// peer; k_scap_merge waits and writes the caller's buffers.  A rank's slice, in uint4 units, for its nw walked pairs
// (dense n_pod * its window's width, else n_pair): [0] header {fault word}, then nw u16 copies padded to 16 bytes, then
// (only when the caller asked for them) nw u8 stops padded to 16 bytes.  A pair's count depends on its own node's state
// alone, so taking each pair from the rank that owns its node gives the single-inventory answer on the world's state for
// any partition.
struct CapMerge {
    const uint4* part;            // this rank's slice; a peer's is at my_stage + sender * slice4
    uint32_t slice4;              // uint4 units of one sender's slice in the exchange
    const uint32_t* cand_nodes; const uint32_t* cand_off;   // cand_off == nullptr: dense form
    uint32_t n_pod, n_pair, n_node;
    uint32_t bounds[PEER_MAX + 1];   // rank r owns nodes [bounds[r], bounds[r + 1])
    const uint32_t* gate;            // this rank's fault word
    uint16_t* pair_copies; uint8_t* pair_stop;                   // the caller's (pair_stop: nullptr unless asked)
    unsigned long long* pod_total; uint32_t* pod_nodes;          // the caller's (each nullptr unless asked)
};

// At most SMs / 4 CTAs, launched after the evaluation: ranks sharing one device must not find their evaluation's SMs
// held by a peer's waiting CTAs.  Block 0 raises this rank's flags, every block waits and checks every rank's fault word;
// then a warp per pod: each lane takes a pair from the slice of the rank owning its node (a candidate naming no node: 0
// copies, POD), writes the pair's outputs and feeds the pod's sums.  Nothing is written after a fault or a timeout.  With
// world 1 (an all-zero PeerExchange) nothing is waited for.
__global__ void __launch_bounds__(256)
k_scap_merge(const PeerExchange x, const CapMerge m) {
    const uint32_t tid = threadIdx.x, world = x.world ? x.world : 1u, rank = x.rank;
    if (!merge_start(x, m.gate, m.slice4, world, rank, tid)) return;
    const uint32_t lane = tid & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + tid) >> 5, n_warp = (gridDim.x * blockDim.x) >> 5;
    const bool dense = m.cand_off == nullptr;
    for (uint32_t p = warp; p < m.n_pod; p += n_warp) {
        unsigned long long k0, k1;
        pod_pairs(m.cand_off, p, m.n_node, 0u, m.n_node, k0, k1);
        cap_pod_sums(p, lane, k0, k1, [&](unsigned long long k) {
            const uint32_t node = pair_node(m.cand_off, m.cand_nodes, k, p, m.n_node);
            uint32_t copies = 0, stop = DRA_ST_POD;                        // a candidate naming no node
            if (node < m.n_node) {
                const uint32_t r = node_owner(m.bounds, world, node);
                const uint32_t lo = m.bounds[r], n_win = m.bounds[r + 1] - lo;
                const uint32_t w = dense ? p * n_win + (node - lo) : (uint32_t)k;
                const uint32_t nw = dense ? m.n_pod * n_win : m.n_pair;
                const uint4* src = r == rank ? m.part : x.my_stage + (size_t)r * m.slice4;
                copies = __ldcg(reinterpret_cast<const unsigned short*>(src + 1) + w);
                if (m.pair_stop) stop = __ldcg(reinterpret_cast<const unsigned char*>(src + 1 + ((size_t)nw + 7) / 8) + w);
            }
            m.pair_copies[k] = (uint16_t)copies;
            if (m.pair_stop) m.pair_stop[k] = (uint8_t)stop;
            return copies;
        }, m.pod_total, m.pod_nodes);
    }
}

}  // namespace dra
