// dra_host.cpp — C++ host layer above the C ABI: the classic-DRA controller.Driver surface
// (Allocate / UnsuitableNodes / Deallocate) with the reference's names.  See include/dra_driver.hpp.
// Lowers strings to flat records, calls libdra_alloc's entry points, lifts OutRecs back to device names.
#include "../../include/dra_driver.hpp"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <stdexcept>

namespace dra {

bool MegabyteMiB(int64_t bytes, uint32_t* mib) {          // limit.Megabyte, sharing.go:234-237
    const int64_t v = bytes / 1024 / 1024;
    if (mib) *mib = v > 0 ? (uint32_t)std::min<int64_t>(v, 0xFFFFFFFFll) : 0;
    return v > 0;
}

std::string CanonicalName(uint32_t gpuIndex) {             // GpuInfo.CanonicalName, deviceinfo.go:74-76
    char b[32]; snprintf(b, sizeof b, "gpu-%u", gpuIndex); return b;
}
std::string CanonicalMigName(uint32_t parentIndex, int32_t giProfileId, uint32_t start, uint32_t size) {
    char b[64]; snprintf(b, sizeof b, "gpu-%u-mig-%d-%u-%u", parentIndex, giProfileId, start, size); return b;   // deviceinfo.go:78-80
}

static const char* status_text(uint8_t st) {
    switch (st) {
        case DRA_ST_NO_CAPACITY: return "no capacity on the selected node";
        case DRA_ST_BAD_PROFILE: return "no GPU on the selected node offers the MIG profile";
        case DRA_ST_GROUP: return "co-located MIG devices do not fit on one parent GPU";
        case DRA_ST_MEM_LIMIT: return "no shareable GPU with enough free memory";
        case DRA_ST_INVALID: return "invalid claim";
        case DRA_ST_POD: return "the pod's claims do not fit on the selected node together";
        case DRA_ST_SEARCH_LIMIT: return "placement search budget exhausted";
        default: return "";
    }
}

Driver::Driver(int cudaDevice) {
    dra_cfg cfg; memset(&cfg, 0, sizeof cfg);
    cfg.abi_version = DRA_ABI_VERSION; cfg.device = cudaDevice;
    int rc = dra_ctx_create(&cfg, &ctx_);
    if (rc != DRA_OK) throw std::runtime_error(std::string("dra_ctx_create: ") + dra_last_error(nullptr));
}
Driver::~Driver() { dra_ctx_destroy(ctx_); }

void Driver::check(int rc, const char* what) {
    if (rc == DRA_OK) return;
    err_ = std::string(what) + ": " + dra_last_error(ctx_);
    throw std::runtime_error(err_);
}

void Driver::SetMigProfiles(uint32_t model, const std::vector<MigProfileInfo>& profiles) {
    dra_profile_tbl t; memset(&t, 0, sizeof t);
    for (const auto& p : profiles) {
        if (p.GiProfileEnum >= DRA_MAX_PROFILES || p.Placements.empty()) continue;
        dra_prof_ent& e = t.ent[p.GiProfileEnum];
        e.size = (uint8_t)p.Placements[0].Size;
        for (const auto& pl : p.Placements) {
            if (pl.Size != e.size) throw std::invalid_argument("placements of one profile differ in size");
            e.start_mask |= (uint16_t)(1u << pl.Start);
        }
    }
    check(dra_set_placement_table(ctx_, model, &t), "dra_set_placement_table");
    profiles_[model] = profiles;
}

void Driver::SetNodes(const std::vector<NodeAllocationState>& nodes) {
    std::vector<dra_gpu_rec> recs;
    nodeIdx_.clear(); nodeName_.clear(); nodeOff_.assign(1, 0); nodeModel_.clear(); gpuLocalIndex_.clear(); held_.clear();
    for (uint32_t n = 0; n < nodes.size(); ++n) {
        nodeIdx_[nodes[n].Node] = n; nodeName_.push_back(nodes[n].Node);
        nodeModel_.push_back(nodes[n].Gpus.empty() ? 0 : nodes[n].Gpus[0].Model);
        for (const auto& g : nodes[n].Gpus) {
            dra_gpu_rec r; memset(&r, 0, sizeof r);
            r.flags = g.MigEnabled ? DRA_GPU_MIG_ENABLED : 0;    // nvlib.go:152 / :316-318
            r.model = (uint8_t)g.Model;
            r.mem_free_mib = (uint32_t)std::min<uint64_t>(g.MemoryBytes >> 20, 0xFFFFFFFFull);
            r.node = n;
            for (const auto& md : g.MigDevices)                   // memorySlice<i>, deviceinfo.go:199-204
                r.busy |= (uint16_t)(((1u << md.second.Size) - 1u) << md.second.Start);
            recs.push_back(r);
            gpuLocalIndex_.push_back(g.Index);
        }
        nodeOff_.push_back((uint32_t)recs.size());
    }
    check(dra_set_inventory(ctx_, recs.data(), (uint32_t)recs.size(), nodeOff_.data(), (uint32_t)nodes.size()), "dra_set_inventory");
}

uint32_t Driver::nodeIndex(const std::string& name) const {
    auto it = nodeIdx_.find(name);
    return it == nodeIdx_.end() ? 0xFFFFFFFFu : it->second;
}

bool Driver::lower(ClaimAllocation& ca, uint32_t node, uint32_t group, Lowered& lo, uint32_t model) {
    ca.Error.clear(); ca.Allocation.clear();
    dra_claim_rec r; memset(&r, 0, sizeof r);
    r.node = node;
    uint32_t copies = 1;
    if (ca.IsMig) {
        r.kind = DRA_KIND_MIG; r.count = 1; r.group = group;
        const auto pit = profiles_.find(model);
        bool found = false;
        if (pit != profiles_.end())
            for (const auto& p : pit->second) if (p.Name == ca.Mig.Profile) { r.profile = (uint8_t)p.GiProfileEnum; found = true; break; }
        if (!found) { ca.Error = "unknown MIG profile '" + ca.Mig.Profile + "'"; return false; }
    } else if (ca.Gpu.Sharing.Strategy == SharingStrategy::None) {
        if (ca.Gpu.Count < 1 || ca.Gpu.Count > DRA_MAX_COUNT) { ca.Error = "count must be in [1, 32]"; return false; }
        r.kind = DRA_KIND_GPU; r.count = (uint16_t)ca.Gpu.Count;
    } else {
        r.kind = DRA_KIND_SHARED; r.count = 1; copies = std::max(1u, ca.Gpu.Count);
        if (ca.Gpu.Sharing.Strategy == SharingStrategy::MPS && ca.Gpu.Sharing.MpsPinnedDeviceMemoryLimitBytes != 0) {
            uint32_t mib = 0;
            if (!MegabyteMiB(ca.Gpu.Sharing.MpsPinnedDeviceMemoryLimitBytes, &mib)) { ca.Error = "invalid limit: value set too low"; return false; }
            r.mem_limit_mib = mib;
        }
    }
    for (uint32_t k = 0; k < copies; ++k) {
        lo.recs.push_back(r); lo.outOff.push_back(lo.nOut); lo.owner.push_back(&ca);
        lo.nOut += r.kind == DRA_KIND_GPU ? r.count : 1;
    }
    return true;
}

void Driver::lift(const Lowered& lo, const std::vector<dra_out_rec>& out, bool commit) {
    // group the records by owning claim (they are contiguous)
    size_t i = 0;
    while (i < lo.recs.size()) {
        ClaimAllocation* ca = lo.owner[i];
        size_t j = i;
        bool ok = true; uint8_t bad = 0;
        Held h;
        while (j < lo.recs.size() && lo.owner[j] == ca) {
            const uint32_t slots = lo.recs[j].kind == DRA_KIND_GPU ? lo.recs[j].count : 1;
            h.recs.push_back(lo.recs[j]); h.outOff.push_back((uint32_t)h.out.size());
            for (uint32_t s = 0; s < slots; ++s) {
                const dra_out_rec& o = out[lo.outOff[j] + s];
                h.out.push_back(o);
                if (o.status != DRA_ST_OK) { ok = false; bad = o.status; }
            }
            ++j;
        }
        if (ok) {
            const uint32_t node = lo.recs[i].node;
            for (const auto& o : h.out) {
                AllocatedDevice d;
                d.GpuIndex = gpuLocalIndex_[o.gpu]; d.Start = o.start; d.Size = o.size;
                if (o.profile < DRA_MAX_PROFILES) {
                    const auto& ps = profiles_[nodeModel_[node]];
                    for (const auto& p : ps) if (p.GiProfileEnum == o.profile) d.GiProfileId = p.GiProfileId;
                    d.Device = CanonicalMigName(d.GpuIndex, d.GiProfileId, d.Start, d.Size);
                } else d.Device = CanonicalName(d.GpuIndex);
                ca->Allocation.push_back(d);
            }
            ca->AllocatedNode = nodeName_[node];
            if (commit) held_[ca->ClaimUID] = h;
        } else {
            ca->Error = status_text(bad);
            // a multi-record claim that failed half-way gives back what it took
            if (commit && h.recs.size() > 1)
                check(dra_deallocate_batch(ctx_, h.recs.data(), (uint32_t)h.recs.size(), h.outOff.data(), h.out.data(), (uint32_t)h.out.size()), "dra_deallocate_batch");
        }
        i = j;
    }
}


// Claims of one pod in lowering order: members of a co-location group (same GpuClaimName) made ADJACENT, in order of
// the group's first appearance.  The device only co-locates CONSECUTIVE claims with equal group (spec §6); members
// separated by another claim would be independent runs that may land on different parents while still reporting
// success — a silent violation of matchAttribute parentUUID (gpu-test4.yaml:42-44).
static std::vector<ClaimAllocation*> groupAdjacent(const std::vector<ClaimAllocation*>& claims) {
    std::vector<std::vector<ClaimAllocation*>> runs;
    std::map<std::string, size_t> runOf;
    for (ClaimAllocation* ca : claims) {
        if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
            auto it = runOf.find(ca->Mig.GpuClaimName);
            if (it != runOf.end()) { runs[it->second].push_back(ca); continue; }
            runOf[ca->Mig.GpuClaimName] = runs.size();
        }
        runs.push_back({ca});
    }
    std::vector<ClaimAllocation*> out;
    for (auto& r : runs) out.insert(out.end(), r.begin(), r.end());
    return out;
}

void Driver::AllocateBatch(const std::vector<PodRequest>& pods) {
    Lowered lo;
    std::vector<uint32_t> podOff(1, 0);                          // pod mode (spec §12): one pod per PodRequest
    for (const auto& pod : pods) {
        const uint32_t node = nodeIndex(pod.SelectedNode);
        std::map<std::string, uint32_t> groups;
        for (ClaimAllocation* ca : groupAdjacent(pod.Claims)) {
            if (node == 0xFFFFFFFFu) { ca->Error = "unknown node '" + pod.SelectedNode + "'"; ca->Allocation.clear(); continue; }
            uint32_t g = 0;
            if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
                auto it = groups.find(ca->Mig.GpuClaimName);
                g = it == groups.end() ? (groups[ca->Mig.GpuClaimName] = nextGroup_++) : it->second;
                if (nextGroup_ == 0) nextGroup_ = 1;
            }
            lower(*ca, node, g, lo, nodeModel_[node]);
        }
        podOff.push_back((uint32_t)lo.recs.size());
    }
    if (lo.recs.empty()) return;
    std::vector<dra_out_rec> out(lo.nOut);
    if (exhaustive_)
        check(dra_allocate_pods_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), podOff.data(), (uint32_t)podOff.size() - 1,
                                      lo.outOff.data(), out.data(), lo.nOut, DRA_F_EXHAUSTIVE), "dra_allocate_pods_batch");
    else
        check(dra_allocate_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), lo.outOff.data(), out.data(), lo.nOut, 0), "dra_allocate_batch");
    lift(lo, out, true);
}

void Driver::Allocate(const std::vector<ClaimAllocation*>& claims, const std::string& selectedNode) {
    PodRequest p; p.Claims = claims; p.SelectedNode = selectedNode;
    AllocateBatch({p});
}

void Driver::UnsuitableNodesBatch(const std::vector<PodRequest>& pods) {
    Lowered lo;
    std::vector<uint32_t> podOff(1, 0), candOff(1, 0), cand;
    std::vector<size_t> podOf;                                  // lowered pod -> index in pods
    for (size_t pi = 0; pi < pods.size(); ++pi) {
        const auto& pod = pods[pi];
        // profile names resolve against the first known candidate's model (homogeneous clusters); a pod whose
        // claims cannot be lowered is unsuitable everywhere
        uint32_t model = 0;
        for (const auto& nn : pod.PotentialNodes) { const uint32_t n = nodeIndex(nn); if (n != 0xFFFFFFFFu) { model = nodeModel_[n]; break; } }
        std::map<std::string, uint32_t> groups;
        bool ok = true;
        const size_t mark = lo.recs.size();
        const uint32_t markOut = lo.nOut;
        for (ClaimAllocation* ca : groupAdjacent(pod.Claims)) {
            uint32_t g = 0;
            if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
                auto it = groups.find(ca->Mig.GpuClaimName);
                g = it == groups.end() ? (groups[ca->Mig.GpuClaimName] = nextGroup_++) : it->second;
                if (nextGroup_ == 0) nextGroup_ = 1;
            }
            ok = lower(*ca, 0, g, lo, model) && ok;
        }
        if (!ok) {
            lo.recs.resize(mark); lo.outOff.resize(mark); lo.owner.resize(mark); lo.nOut = markOut;
            for (ClaimAllocation* ca : pod.Claims) for (const auto& nn : pod.PotentialNodes) ca->UnsuitableNodes.push_back(nn);
            continue;
        }
        podOff.push_back((uint32_t)lo.recs.size());
        for (const auto& nn : pod.PotentialNodes) cand.push_back(nodeIndex(nn));
        candOff.push_back((uint32_t)cand.size());
        podOf.push_back(pi);
    }
    if (podOf.empty()) return;
    std::vector<uint8_t> bits((cand.size() + 7) / 8 + 1, 0);
    check(dra_unsuitable_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), podOff.data(), (uint32_t)podOf.size(),
                               cand.data(), candOff.data(), bits.data(), exhaustive_ ? DRA_F_EXHAUSTIVE : 0u), "dra_unsuitable_batch");
    for (size_t q = 0; q < podOf.size(); ++q) {
        const auto& pod = pods[podOf[q]];
        for (uint32_t k = candOff[q]; k < candOff[q + 1]; ++k) {
            if ((bits[k >> 3] >> (k & 7)) & 1) continue;
            // all-or-nothing per pod: the node goes to EVERY claim's UnsuitableNodes (SURVEY App. A)
            for (ClaimAllocation* ca : pod.Claims) ca->UnsuitableNodes.push_back(pod.PotentialNodes[k - candOff[q]]);
        }
    }
}

void Driver::PlaceBatch(const std::vector<PodRequest>& pods) {
    Lowered lo;
    std::vector<uint32_t> podOff(1, 0), candOff(1, 0), cand;
    std::vector<size_t> podOf;                                  // lowered pod -> index in pods
    for (size_t pi = 0; pi < pods.size(); ++pi) {
        const auto& pod = pods[pi];
        // profile names resolve against the first known candidate's model, as in UnsuitableNodesBatch; a pod whose
        // claims cannot be lowered is not placed (each claim's Error says why)
        uint32_t model = 0;
        for (const auto& nn : pod.PotentialNodes) { const uint32_t n = nodeIndex(nn); if (n != 0xFFFFFFFFu) { model = nodeModel_[n]; break; } }
        std::map<std::string, uint32_t> groups;
        bool ok = true;
        const size_t mark = lo.recs.size();
        const uint32_t markOut = lo.nOut;
        for (ClaimAllocation* ca : groupAdjacent(pod.Claims)) {
            uint32_t g = 0;
            if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
                auto it = groups.find(ca->Mig.GpuClaimName);
                g = it == groups.end() ? (groups[ca->Mig.GpuClaimName] = nextGroup_++) : it->second;
                if (nextGroup_ == 0) nextGroup_ = 1;
            }
            ca->AllocatedNode.clear();
            ok = lower(*ca, 0, g, lo, model) && ok;             // node: ignored by the call, set from its answer below
        }
        if (!ok) {
            lo.recs.resize(mark); lo.outOff.resize(mark); lo.owner.resize(mark); lo.nOut = markOut;
            continue;
        }
        podOff.push_back((uint32_t)lo.recs.size());
        for (const auto& nn : pod.PotentialNodes) cand.push_back(nodeIndex(nn));
        candOff.push_back((uint32_t)cand.size());
        podOf.push_back(pi);
    }
    if (podOf.empty()) return;
    std::vector<dra_out_rec> out(lo.nOut);
    std::vector<uint32_t> podNode(podOf.size());
    check(dra_place_pods_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), podOff.data(), (uint32_t)podOf.size(),
                               cand.data(), candOff.data(), lo.outOff.data(), out.data(), lo.nOut, podNode.data(),
                               exhaustive_ ? DRA_F_EXHAUSTIVE : 0u), "dra_place_pods_batch");
    for (size_t q = 0; q < podOf.size(); ++q)                   // the records name the chosen node: lift and Deallocate need it
        for (uint32_t i = podOff[q]; i < podOff[q + 1]; ++i) lo.recs[i].node = podNode[q] == DRA_GPU_NONE ? 0u : podNode[q];
    lift(lo, out, true);
    for (size_t q = 0; q < podOf.size(); ++q)
        if (podNode[q] == DRA_GPU_NONE)
            for (ClaimAllocation* ca : pods[podOf[q]].Claims)
                if (ca->Error == status_text(DRA_ST_POD)) ca->Error = "the pod's claims fit together on none of its potential nodes";
}

std::vector<std::map<std::string, uint32_t>> Driver::PodCapacityBatch(const std::vector<PodRequest>& pods, uint32_t maxCopies) {
    std::vector<std::map<std::string, uint32_t>> res(pods.size());
    Lowered lo;
    std::vector<uint32_t> podOff(1, 0), candOff(1, 0), cand;
    std::vector<size_t> podOf;                                  // lowered pod -> index in pods
    for (size_t pi = 0; pi < pods.size(); ++pi) {
        const auto& pod = pods[pi];
        uint32_t model = 0;                                     // profile names: as in UnsuitableNodesBatch
        for (const auto& nn : pod.PotentialNodes) { const uint32_t n = nodeIndex(nn); if (n != 0xFFFFFFFFu) { model = nodeModel_[n]; break; } }
        std::map<std::string, uint32_t> groups;
        bool ok = true;
        const size_t mark = lo.recs.size();
        const uint32_t markOut = lo.nOut;
        for (ClaimAllocation* ca : groupAdjacent(pod.Claims)) {
            uint32_t g = 0;
            if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
                auto it = groups.find(ca->Mig.GpuClaimName);
                g = it == groups.end() ? (groups[ca->Mig.GpuClaimName] = nextGroup_++) : it->second;
                if (nextGroup_ == 0) nextGroup_ = 1;
            }
            ok = lower(*ca, 0, g, lo, model) && ok;
        }
        if (!ok) {
            lo.recs.resize(mark); lo.outOff.resize(mark); lo.owner.resize(mark); lo.nOut = markOut;
            continue;
        }
        podOff.push_back((uint32_t)lo.recs.size());
        for (const auto& nn : pod.PotentialNodes) cand.push_back(nodeIndex(nn));
        candOff.push_back((uint32_t)cand.size());
        podOf.push_back(pi);
    }
    if (podOf.empty()) return res;
    std::vector<uint16_t> copies(cand.size() + 1, 0);
    check(dra_pod_capacity_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), podOff.data(), (uint32_t)podOf.size(),
                                 cand.data(), candOff.data(), maxCopies, copies.data(), nullptr, nullptr, nullptr,
                                 exhaustive_ ? DRA_F_EXHAUSTIVE : 0u), "dra_pod_capacity_batch");
    for (size_t q = 0; q < podOf.size(); ++q)
        for (uint32_t k = candOff[q]; k < candOff[q + 1]; ++k)
            res[podOf[q]][pods[podOf[q]].PotentialNodes[k - candOff[q]]] = copies[k];
    return res;
}

// "1 node" / "2 nodes"
static std::string nodes_text(size_t n) { return std::to_string(n) + (n == 1 ? " node" : " nodes"); }

static const char* why_text(uint8_t r) {
    switch (r) {
        case DRA_ST_NO_CAPACITY: return "no capacity";
        case DRA_ST_BAD_PROFILE: return "no GPU offers the MIG profile";
        case DRA_ST_GROUP: return "co-located MIG devices do not fit on one parent GPU";
        case DRA_ST_MEM_LIMIT: return "no shareable GPU with enough free memory";
        case DRA_ST_INVALID: return "invalid claim";
        case DRA_ST_POD: return "does not fit together with the pod's other claims";
        case DRA_ST_SEARCH_LIMIT: return "placement search budget exhausted";
        default: return "";
    }
}

// `claim "uid" (MIG 3g.20gb)`, `claim "uid" (2 GPUs)`, `claim "uid" (shared GPU)`
static std::string claim_text(const ClaimAllocation& ca) {
    std::string what;
    if (ca.IsMig) what = "MIG " + ca.Mig.Profile;
    else if (ca.Gpu.Sharing.Strategy == SharingStrategy::None) what = std::to_string(ca.Gpu.Count) + (ca.Gpu.Count == 1 ? " GPU" : " GPUs");
    else what = "shared GPU";
    return "claim \"" + ca.ClaimUID + "\" (" + what + ")";
}

// One pod's message from its pairs [k0, k1): "2/5 nodes are available: 2 nodes: claim ... no capacity; 1 node: ...",
// nodes grouped by (reason, blocking claim), largest group first, ties in pair order.  The blocking claim is an index
// into the LOWERED records: owner maps it back (group members were made adjacent, so it is not the position in
// pod.Claims).
static std::string why_message(const std::vector<ClaimAllocation*>& owner, const uint8_t* why, const uint32_t* blk,
                               uint32_t k0, uint32_t k1) {
    std::vector<std::pair<std::string, size_t>> parts;          // text, nodes; in order of first appearance
    std::map<std::string, size_t> at;
    size_t ok = 0;
    for (uint32_t k = k0; k < k1; ++k) {
        if (why[k] == DRA_ST_OK) { ++ok; continue; }
        std::string t;
        if (why[k] == DRA_WHY_NO_NODE) t = "not in the inventory";
        else if (blk[k] == DRA_WHY_CLAIM_NONE) t = std::string("more than ") + std::to_string(DRA_MAX_POD) + " claims";
        else t = claim_text(*owner[blk[k]]) + " " + why_text(why[k]);
        auto it = at.find(t);
        if (it == at.end()) { at[t] = parts.size(); parts.push_back({t, 1}); } else ++parts[it->second].second;
    }
    std::stable_sort(parts.begin(), parts.end(), [](const auto& a, const auto& b) { return a.second > b.second; });
    std::string m = std::to_string(ok) + "/" + std::to_string(k1 - k0) + " nodes are available";
    for (size_t i = 0; i < parts.size(); ++i) m += (i ? "; " : ": ") + nodes_text(parts[i].second) + ": " + parts[i].first;
    return m + ".";
}

// The message of a pod whose claims cannot be lowered: its first such claim and that claim's Error
static std::string unlowered_message(const Driver::PodRequest& pod) {
    const size_t n = pod.PotentialNodes.size();
    for (ClaimAllocation* ca : pod.Claims)
        if (!ca->Error.empty())
            return "0/" + std::to_string(n) + " nodes are available" + (n ? ": " + nodes_text(n) + ": " + claim_text(*ca) + " " + ca->Error : "") + ".";
    return "";
}

std::vector<std::string> Driver::UnsuitableReasonsBatch(const std::vector<PodRequest>& pods) {
    std::vector<std::string> res(pods.size());
    Lowered lo;
    std::vector<uint32_t> podOff(1, 0), candOff(1, 0), cand;
    std::vector<size_t> podOf;                                  // lowered pod -> index in pods
    for (size_t pi = 0; pi < pods.size(); ++pi) {
        const auto& pod = pods[pi];
        uint32_t model = 0;                                     // profile names: as in UnsuitableNodesBatch
        for (const auto& nn : pod.PotentialNodes) { const uint32_t n = nodeIndex(nn); if (n != 0xFFFFFFFFu) { model = nodeModel_[n]; break; } }
        std::map<std::string, uint32_t> groups;
        bool ok = true;
        const size_t mark = lo.recs.size();
        const uint32_t markOut = lo.nOut;
        for (ClaimAllocation* ca : groupAdjacent(pod.Claims)) {
            uint32_t g = 0;
            if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
                auto it = groups.find(ca->Mig.GpuClaimName);
                g = it == groups.end() ? (groups[ca->Mig.GpuClaimName] = nextGroup_++) : it->second;
                if (nextGroup_ == 0) nextGroup_ = 1;
            }
            ok = lower(*ca, 0, g, lo, model) && ok;
        }
        if (!ok) {
            lo.recs.resize(mark); lo.outOff.resize(mark); lo.owner.resize(mark); lo.nOut = markOut;
            res[pi] = unlowered_message(pod);
            continue;
        }
        podOff.push_back((uint32_t)lo.recs.size());
        for (const auto& nn : pod.PotentialNodes) cand.push_back(nodeIndex(nn));
        candOff.push_back((uint32_t)cand.size());
        podOf.push_back(pi);
    }
    if (podOf.empty()) return res;
    std::vector<uint8_t> why(cand.size() + 1, 0);
    std::vector<uint32_t> blk(cand.size() + 1, 0);
    check(dra_unsuitable_why_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), podOff.data(), (uint32_t)podOf.size(),
                                   cand.data(), candOff.data(), why.data(), blk.data(), nullptr, nullptr,
                                   exhaustive_ ? DRA_F_EXHAUSTIVE : 0u), "dra_unsuitable_why_batch");
    for (size_t q = 0; q < podOf.size(); ++q) res[podOf[q]] = why_message(lo.owner, why.data(), blk.data(), candOff[q], candOff[q + 1]);
    return res;
}

std::vector<std::string> Driver::PlaceBatchWithReasons(const std::vector<PodRequest>& pods) {
    std::vector<std::string> res(pods.size());
    Lowered lo;
    std::vector<uint32_t> podOff(1, 0), candOff(1, 0), cand;
    std::vector<size_t> podOf;                                  // lowered pod -> index in pods
    for (size_t pi = 0; pi < pods.size(); ++pi) {
        const auto& pod = pods[pi];
        uint32_t model = 0;                                     // profile names: as in PlaceBatch
        for (const auto& nn : pod.PotentialNodes) { const uint32_t n = nodeIndex(nn); if (n != 0xFFFFFFFFu) { model = nodeModel_[n]; break; } }
        std::map<std::string, uint32_t> groups;
        bool ok = true;
        const size_t mark = lo.recs.size();
        const uint32_t markOut = lo.nOut;
        for (ClaimAllocation* ca : groupAdjacent(pod.Claims)) {
            uint32_t g = 0;
            if (ca->IsMig && !ca->Mig.GpuClaimName.empty()) {
                auto it = groups.find(ca->Mig.GpuClaimName);
                g = it == groups.end() ? (groups[ca->Mig.GpuClaimName] = nextGroup_++) : it->second;
                if (nextGroup_ == 0) nextGroup_ = 1;
            }
            ca->AllocatedNode.clear();
            ok = lower(*ca, 0, g, lo, model) && ok;
        }
        if (!ok) {
            lo.recs.resize(mark); lo.outOff.resize(mark); lo.owner.resize(mark); lo.nOut = markOut;
            res[pi] = unlowered_message(pod);
            continue;
        }
        podOff.push_back((uint32_t)lo.recs.size());
        for (const auto& nn : pod.PotentialNodes) cand.push_back(nodeIndex(nn));
        candOff.push_back((uint32_t)cand.size());
        podOf.push_back(pi);
    }
    if (podOf.empty()) return res;
    std::vector<dra_out_rec> out(lo.nOut);
    std::vector<uint32_t> podNode(podOf.size());
    std::vector<uint8_t> why(cand.size() + 1, 0);
    std::vector<uint32_t> blk(cand.size() + 1, 0);
    check(dra_place_pods_why_batch(ctx_, lo.recs.data(), (uint32_t)lo.recs.size(), podOff.data(), (uint32_t)podOf.size(),
                                   cand.data(), candOff.data(), lo.outOff.data(), out.data(), lo.nOut, podNode.data(),
                                   why.data(), blk.data(), nullptr, nullptr, exhaustive_ ? DRA_F_EXHAUSTIVE : 0u),
          "dra_place_pods_why_batch");
    for (size_t q = 0; q < podOf.size(); ++q) res[podOf[q]] = why_message(lo.owner, why.data(), blk.data(), candOff[q], candOff[q + 1]);
    for (size_t q = 0; q < podOf.size(); ++q)                   // from here on as PlaceBatch
        for (uint32_t i = podOff[q]; i < podOff[q + 1]; ++i) lo.recs[i].node = podNode[q] == DRA_GPU_NONE ? 0u : podNode[q];
    lift(lo, out, true);
    for (size_t q = 0; q < podOf.size(); ++q)
        if (podNode[q] == DRA_GPU_NONE)
            for (ClaimAllocation* ca : pods[podOf[q]].Claims)
                if (ca->Error == status_text(DRA_ST_POD)) ca->Error = "the pod's claims fit together on none of its potential nodes";
    return res;
}

void Driver::UnsuitableNodes(const std::vector<ClaimAllocation*>& claims, const std::vector<std::string>& potentialNodes) {
    PodRequest p; p.Claims = claims; p.PotentialNodes = potentialNodes;
    UnsuitableNodesBatch({p});
}

void Driver::Deallocate(ClaimAllocation& claim) {
    auto it = held_.find(claim.ClaimUID);
    if (it == held_.end()) return;                              // idempotent, like Unprepare (device_state.go:171-173)
    Held& h = it->second;
    check(dra_deallocate_batch(ctx_, h.recs.data(), (uint32_t)h.recs.size(), h.outOff.data(), h.out.data(), (uint32_t)h.out.size()), "dra_deallocate_batch");
    held_.erase(it);
    claim.Allocation.clear(); claim.AllocatedNode.clear();
}

uint16_t Driver::BusyMask(const std::string& node, uint32_t gpuIndex) {
    const uint32_t n = nodeIndex(node);
    if (n == 0xFFFFFFFFu) return 0;
    std::vector<dra_gpu_rec> inv(nodeOff_.back());
    check(dra_get_inventory(ctx_, inv.data(), (uint32_t)inv.size()), "dra_get_inventory");
    for (uint32_t g = nodeOff_[n]; g < nodeOff_[n + 1]; ++g) if (gpuLocalIndex_[g] == gpuIndex) return inv[g].busy;
    return 0;
}

}  // namespace dra
