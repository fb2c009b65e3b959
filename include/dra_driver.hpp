// dra_driver.hpp — C++ host side above the C ABI (include/dra_alloc.h).
//
// The reference is Go; Go is not installed in this image, so the host layer a Go driver would put above the
// cgo calls is written here in C++ with the reference's own names and argument meaning:
//
//   * Driver::Allocate / UnsuitableNodes / Deallocate   — the classic-DRA `controller.Driver` surface that
//     BASELINE.json's north_star names (k8s.io/dynamic-resource-allocation/controller; removed from the
//     snapshot, SURVEY.md F1).  Per-claim failures are reported in ClaimAllocation::Error, never thrown —
//     like the per-claim Error strings of cmd/nvidia-dra-plugin/driver.go:126-137.
//   * GpuClaimParametersSpec / MigDeviceClaimParametersSpec — the legacy claim parameter shapes
//     (demo/specs/selectors/parameters.yaml:7-27, demo/specs/mig+mps/sharing-demo-parameters.yaml:22-41).
//   * AllocatableGpu / MigPlacement — GpuInfo + MigDevicePlacement of cmd/nvidia-dra-plugin/deviceinfo.go:30-64.
//   * device names  gpu-<index>  /  gpu-<parentIndex>-mig-<profileId>-<start>-<size>  — deviceinfo.go:74-80.
//
// Everything that decides an allocation happens in libdra_alloc.so's kernels; this layer only lowers
// strings to flat records and lifts OutRecs back to names.
#pragma once

#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "dra_alloc.h"

namespace dra {

enum class SharingStrategy { None, TimeSlicing, MPS };          // sharing.go:30-35

struct GpuSharing {                                             // sharing.go:63-67 (the fields allocation needs)
    SharingStrategy Strategy = SharingStrategy::None;
    int64_t MpsPinnedDeviceMemoryLimitBytes = 0;                // MpsConfig.DefaultPinnedDeviceMemoryLimit.Value()
};

struct GpuClaimParametersSpec {                                 // legacy GpuClaimParameters.spec
    uint32_t Count = 1;
    GpuSharing Sharing;
};

struct MigDeviceClaimParametersSpec {                           // legacy MigDeviceClaimParameters.spec
    std::string Profile;                                        // "1g.5gb", "3g.20gb", ... (go-nvlib mig_profile.go:145-154)
    std::string GpuClaimName;                                   // co-location key: claims sharing it share a parent GPU
};

struct AllocatedDevice {                                        // one DeviceRequestAllocationResult (k8s types.go:795-840)
    std::string Device;                                         // canonical name, deviceinfo.go:74-80
    uint32_t GpuIndex = 0;                                      // index on the node
    uint32_t Start = 0, Size = 0;
    int32_t GiProfileId = -1;
};

struct ClaimAllocation {                                        // controller.ClaimAllocation
    std::string ClaimUID;
    bool IsMig = false;
    GpuClaimParametersSpec Gpu;
    MigDeviceClaimParametersSpec Mig;
    // results
    std::vector<std::string> UnsuitableNodes;
    std::vector<AllocatedDevice> Allocation;
    std::string Error;                                          // empty = allocated
    std::string AllocatedNode;
};

struct MigPlacement { uint32_t Start, Size; };                  // nvml.GpuInstancePlacement, types_gen.go:755-758

struct MigProfileInfo {                                         // deviceinfo.go:57-60 + nvml profile id
    std::string Name;                                           // "1g.5gb"
    uint32_t GiProfileEnum;                                     // nvml GPU_INSTANCE_PROFILE_* 0..9 (const.go:745-766)
    int32_t GiProfileId;                                        // GpuInstanceProfileInfo.Id, used in device names
    std::vector<MigPlacement> Placements;                       // GetGpuInstancePossiblePlacements, nvlib.go:257-274
};

struct AllocatableGpu {                                         // GpuInfo, deviceinfo.go:30-43
    uint32_t Index = 0;
    bool MigEnabled = false;
    uint64_t MemoryBytes = 0;
    uint32_t Model = 0;                                         // placement-table row
    std::vector<std::pair<std::string, MigPlacement>> MigDevices;   // existing MIG devices: profile name, placement
};

struct NodeAllocationState {                                    // per-node view (classic CRD / one ResourceSlice pool)
    std::string Node;
    std::vector<AllocatableGpu> Gpus;                           // ordered by Index
};

class Driver {
public:
    explicit Driver(int cudaDevice = 0);
    ~Driver();
    Driver(const Driver&) = delete;
    Driver& operator=(const Driver&) = delete;

    // model = row of the placement table; profiles as enumerated by getGpuInfo (nvlib.go:244-295)
    void SetMigProfiles(uint32_t model, const std::vector<MigProfileInfo>& profiles);
    // replaces the whole inventory (publish / NAS sync)
    void SetNodes(const std::vector<NodeAllocationState>& nodes);
    // spec §12: evaluate each pod atomically, its MIG claims by the backtracking search over every valid placement
    // (the classic mig.allocate, SURVEY App. A) instead of in-order first-fit.  Off by default.
    void SetExhaustive(bool on) { exhaustive_ = on; }

    // controller.Driver.Allocate(ctx, claims, selectedNode): mutates the inventory
    void Allocate(const std::vector<ClaimAllocation*>& claims, const std::string& selectedNode);
    // controller.Driver.UnsuitableNodes(ctx, pod, claims, potentialNodes): appends to every claim's
    // UnsuitableNodes the nodes on which the pod's claims cannot all be satisfied; pure
    void UnsuitableNodes(const std::vector<ClaimAllocation*>& claims, const std::vector<std::string>& potentialNodes);
    // controller.Driver.Deallocate(ctx, claim)
    void Deallocate(ClaimAllocation& claim);

    // batched forms (many pods per call) — what the kernels are built for
    struct PodRequest { std::vector<ClaimAllocation*> Claims; std::string SelectedNode; std::vector<std::string> PotentialNodes; };
    void AllocateBatch(const std::vector<PodRequest>& pods);
    void UnsuitableNodesBatch(const std::vector<PodRequest>& pods);
    // choose the node and allocate in one call (spec §13, dra_place_pods_batch): pods in order, each on the first of its
    // PotentialNodes where all its claims fit, given what the pods before it took — the classic controller's pending
    // allocations.  SelectedNode is not read; each claim gets AllocatedNode and Allocation, or Error when the pod fits
    // on none of its nodes.  Each pod is atomic (spec §12), its MIG claims by the backtracking search when
    // SetExhaustive(true).  Placed claims can be given back with Deallocate.
    void PlaceBatch(const std::vector<PodRequest>& pods);
    // how many copies of each pod every one of its PotentialNodes still takes (spec §16, dra_pod_capacity_batch), counted
    // as AllocateBatch would place them under SetExhaustive, at most maxCopies (1 .. 65535) per node; pure.  Result q:
    // node name -> copies for pod q; a node the inventory does not know counts 0, and a pod whose claims cannot be
    // lowered gets an empty map (each claim's Error says why).  SelectedNode is not read.
    std::vector<std::map<std::string, uint32_t>> PodCapacityBatch(const std::vector<PodRequest>& pods, uint32_t maxCopies);
    // why each pod fits none, some or all of its PotentialNodes (spec §17, dra_unsuitable_why_batch), as kube-scheduler's
    // FitError says it: one message per pod, e.g. `0/3 nodes are available: 2 nodes: claim "c1" (MIG 3g.20gb) no
    // capacity; 1 node: not in the inventory.`  Nodes are grouped by (reason, blocking claim), largest group first, ties
    // in the order of PotentialNodes; claims are named by ClaimUID.  Judged as UnsuitableNodesBatch judges them under
    // SetExhaustive; pure.  A pod whose claims cannot be lowered names its first such claim and its Error.
    std::vector<std::string> UnsuitableReasonsBatch(const std::vector<PodRequest>& pods);
    // PlaceBatch that also says why each pod went where it did, or nowhere (spec §18, dra_place_pods_why_batch): places
    // exactly as PlaceBatch, setting the same AllocatedNode, Allocation and Error on the claims, and returns one message
    // per pod in UnsuitableReasonsBatch's format, each node judged as the pod met it, after the pods before it.
    std::vector<std::string> PlaceBatchWithReasons(const std::vector<PodRequest>& pods);

    // live occupancy of one GPU (memory-slice mask), for inspection
    uint16_t BusyMask(const std::string& node, uint32_t gpuIndex);
    const std::string& LastError() const { return err_; }

private:
    struct Lowered { std::vector<dra_claim_rec> recs; std::vector<uint32_t> outOff; std::vector<ClaimAllocation*> owner; uint32_t nOut = 0; };
    bool lower(ClaimAllocation& ca, uint32_t node, uint32_t group, Lowered& lo, uint32_t model);
    void lift(const Lowered& lo, const std::vector<dra_out_rec>& out, bool commit);
    uint32_t nodeIndex(const std::string& name) const;
    void check(int rc, const char* what);

    dra_ctx* ctx_ = nullptr;
    std::string err_;
    std::map<std::string, uint32_t> nodeIdx_;
    std::vector<std::string> nodeName_;
    std::vector<uint32_t> nodeOff_;
    std::vector<uint32_t> nodeModel_;                           // model of the node's first GPU (profile-name lookup)
    std::vector<uint32_t> gpuLocalIndex_;                       // GpuInfo.index per global gpu
    std::map<uint32_t, std::vector<MigProfileInfo>> profiles_;  // per model
    uint32_t nextGroup_ = 1;
    bool exhaustive_ = false;
    // what Deallocate needs to undo a claim
    struct Held { std::vector<dra_claim_rec> recs; std::vector<uint32_t> outOff; std::vector<dra_out_rec> out; };
    std::map<std::string, Held> held_;
};

// sharing.go:234-237  limit.Megabyte(): bytes/1024/1024, valid iff > 0
bool MegabyteMiB(int64_t bytes, uint32_t* mib);
// deviceinfo.go:74-80
std::string CanonicalName(uint32_t gpuIndex);
std::string CanonicalMigName(uint32_t parentIndex, int32_t giProfileId, uint32_t start, uint32_t size);

}  // namespace dra
