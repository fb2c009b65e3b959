// place_test.cpp — exercises Driver::PlaceBatch of the C++ host layer (include/dra_driver.hpp): choosing the node and
// allocating in one call, with the pending allocations of the pods before.  Needs an H100.
// Built by k8s-dra-driver_b200/build.py into tests/cpp/place_test; run by tests/test_gpu_place_pods.py.
#include <cstdio>
#include <string>
#include <vector>

#include "dra_driver.hpp"

using namespace dra;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); ++failures; } } while (0)
#define EXPECT_EQ_S(a, b) do { std::string a_ = (a), b_ = (b); if (a_ != b_) { printf("FAIL %s:%d  %s == %s  ('%s' vs '%s')\n", __FILE__, __LINE__, #a, #b, a_.c_str(), b_.c_str()); ++failures; } } while (0)

static std::vector<MigProfileInfo> a100() {          // synthetic A100-40GB table (spec appendix)
    auto pl = [](std::initializer_list<uint32_t> starts, uint32_t size) { std::vector<MigPlacement> v; for (auto s : starts) v.push_back({s, size}); return v; };
    return {
        {"1g.5gb", 0, 19, pl({0, 1, 2, 3, 4, 5, 6}, 1)},
        {"2g.10gb", 1, 14, pl({0, 2, 4}, 2)},
        {"3g.20gb", 2, 9, pl({0, 4}, 4)},
        {"4g.20gb", 3, 5, pl({0}, 4)},
        {"7g.40gb", 4, 0, pl({0}, 8)},
    };
}

static NodeAllocationState node(const std::string& name, int nMig, int nFull) {
    NodeAllocationState n; n.Node = name;
    for (int i = 0; i < nMig + nFull; ++i) { AllocatableGpu g; g.Index = i; g.MigEnabled = i < nMig; g.MemoryBytes = 40ull << 30; n.Gpus.push_back(g); }
    return n;
}

static ClaimAllocation mig(const std::string& uid, const std::string& profile, const std::string& gpuClaim = "") {
    ClaimAllocation c; c.ClaimUID = uid; c.IsMig = true; c.Mig.Profile = profile; c.Mig.GpuClaimName = gpuClaim; return c;
}
static ClaimAllocation gpu(const std::string& uid, uint32_t count = 1) {
    ClaimAllocation c; c.ClaimUID = uid; c.Gpu.Count = count; return c;
}

int main() {
    Driver d(0);
    d.SetMigProfiles(0, a100());
    d.SetNodes({node("node-a", 1, 0), node("node-b", 1, 0), node("node-c", 0, 2)});

    // two pods that each need a whole MIG GPU, both listing node-a first: UnsuitableNodes says node-a fits both,
    // PlaceBatch sends the second to node-b
    {
        auto a = mig("p0", "7g.40gb"), b = mig("p1", "7g.40gb");
        Driver::PodRequest p0, p1;
        p0.Claims = {&a}; p0.PotentialNodes = {"node-a", "node-b"};
        p1.Claims = {&b}; p1.PotentialNodes = {"node-a", "node-b"};
        d.UnsuitableNodesBatch({p0, p1});
        EXPECT(a.UnsuitableNodes.empty() && b.UnsuitableNodes.empty());
        d.PlaceBatch({p0, p1});
        EXPECT(a.Error.empty() && b.Error.empty());
        EXPECT_EQ_S(a.AllocatedNode, "node-a");
        EXPECT_EQ_S(b.AllocatedNode, "node-b");
        EXPECT_EQ_S(a.Allocation.size() == 1 ? a.Allocation[0].Device : "", "gpu-0-mig-0-0-8");
        EXPECT(d.BusyMask("node-a", 0) == 0xFF && d.BusyMask("node-b", 0) == 0xFF);
        // a third pod finds no room anywhere: an error, nothing taken
        auto c = mig("p2", "1g.5gb");
        Driver::PodRequest p2; p2.Claims = {&c}; p2.PotentialNodes = {"node-a", "node-b", "no-such-node"};
        d.PlaceBatch({p2});
        EXPECT(!c.Error.empty() && c.AllocatedNode.empty() && c.Allocation.empty());
        // Deallocate gives the devices back; the next pod can take node-a again
        d.Deallocate(a);
        EXPECT(d.BusyMask("node-a", 0) == 0);
        d.PlaceBatch({p2});
        EXPECT(c.Error.empty());
        EXPECT_EQ_S(c.AllocatedNode, "node-a");
        d.Deallocate(b); d.Deallocate(c);
        EXPECT(d.BusyMask("node-a", 0) == 0 && d.BusyMask("node-b", 0) == 0);
    }
    // a pod of a full GPU and a co-located MIG pair skips the nodes that cannot take all of it
    {
        auto g = gpu("q-gpu", 2);
        Driver::PodRequest p; p.Claims = {&g}; p.PotentialNodes = {"node-a", "node-b", "node-c"};
        d.PlaceBatch({p});
        EXPECT(g.Error.empty());
        EXPECT_EQ_S(g.AllocatedNode, "node-c");
        EXPECT(g.Allocation.size() == 2);
        auto m1 = mig("q-m1", "3g.20gb", "pair"), m2 = mig("q-m2", "3g.20gb", "pair");
        Driver::PodRequest q; q.Claims = {&m1, &m2}; q.PotentialNodes = {"node-c", "node-b"};
        d.PlaceBatch({q});
        EXPECT(m1.Error.empty() && m2.Error.empty());
        EXPECT_EQ_S(m1.AllocatedNode, "node-b");
        EXPECT(m1.Allocation.size() == 1 && m2.Allocation.size() == 1 && m1.Allocation[0].GpuIndex == m2.Allocation[0].GpuIndex);
        d.Deallocate(g); d.Deallocate(m1); d.Deallocate(m2);
        EXPECT(d.BusyMask("node-b", 0) == 0);
    }
    if (failures) { printf("%d failures\n", failures); return 1; }
    printf("place_test ok\n");
    return 0;
}
