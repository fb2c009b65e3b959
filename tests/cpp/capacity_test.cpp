// capacity_test.cpp — exercises Driver::PodCapacityBatch of the C++ host layer (include/dra_driver.hpp): how many copies
// of a pod each of its potential nodes still takes.  Needs an H100.
// Built by k8s-dra-driver_b200/build.py into tests/cpp/capacity_test; run by tests/test_gpu_pod_capacity.py.
#include <cstdio>
#include <string>
#include <vector>

#include "dra_driver.hpp"

using namespace dra;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); ++failures; } } while (0)

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
    d.SetNodes({node("node-a", 1, 0), node("node-b", 4, 0), node("node-c", 0, 2)});
    const std::vector<std::string> all = {"node-a", "node-b", "node-c", "node-x"};

    auto g3 = mig("p0", "3g.20gb"), whole = gpu("p1", 2), bad = mig("p2", "9g.99gb");
    // gpu-test4.yaml: {1g, 1g, 2g, 3g} on one parent GPU
    auto t0 = mig("t0", "1g.5gb", "shared"), t1 = mig("t1", "1g.5gb", "shared"), t2 = mig("t2", "2g.10gb", "shared"),
         t3 = mig("t3", "3g.20gb", "shared");
    Driver::PodRequest p0, p1, p2, p3;
    p0.Claims = {&g3}; p0.PotentialNodes = all;
    p1.Claims = {&whole}; p1.PotentialNodes = all;
    p2.Claims = {&bad}; p2.PotentialNodes = all;
    p3.Claims = {&t0, &t1, &t2, &t3}; p3.PotentialNodes = {"node-b", "node-a"};
    for (bool exhaustive : {false, true}) {
        d.SetExhaustive(exhaustive);
        auto r = d.PodCapacityBatch({p0, p1, p2, p3}, 64);
        EXPECT(r.size() == 4);
        EXPECT(r[0].size() == 4 && r[0]["node-a"] == 2 && r[0]["node-b"] == 8 && r[0]["node-c"] == 0 && r[0]["node-x"] == 0);
        EXPECT(r[1]["node-a"] == 0 && r[1]["node-b"] == 0 && r[1]["node-c"] == 1);
        EXPECT(r[2].empty() && !bad.Error.empty());
        EXPECT(r[3].size() == 2 && r[3]["node-b"] == 4 && r[3]["node-a"] == 1);
        EXPECT(d.PodCapacityBatch({p0}, 3)[0]["node-b"] == 3);               // the cap
        EXPECT(d.BusyMask("node-a", 0) == 0 && d.BusyMask("node-b", 3) == 0);   // pure
    }
    // the count is what Allocate then places: two 3g pods fit node-a, a third does not, and the count follows the inventory
    auto a = mig("a", "3g.20gb"), b = mig("b", "3g.20gb"), c = mig("c", "3g.20gb");
    d.Allocate({&a}, "node-a");
    EXPECT(a.Error.empty() && d.PodCapacityBatch({p0}, 64)[0]["node-a"] == 1);
    d.Allocate({&b}, "node-a");
    EXPECT(b.Error.empty() && d.PodCapacityBatch({p0}, 64)[0]["node-a"] == 0);
    d.Allocate({&c}, "node-a");
    EXPECT(!c.Error.empty());

    if (failures) { printf("capacity_test: %d failure(s)\n", failures); return 1; }
    printf("capacity_test ok\n");
    return 0;
}
