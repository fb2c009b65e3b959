// place_why_test.cpp — exercises Driver::PlaceBatchWithReasons of the C++ host layer (include/dra_driver.hpp): one
// kube-scheduler-style message per pod, each node judged in the state the pod met it, and the same placement as
// PlaceBatch.  Needs an H100.  Built by k8s-dra-driver_b200/build.py into tests/cpp/place_why_test; run by
// tests/test_gpu_place_why.py.
#include <cstdio>
#include <string>
#include <vector>

#include "dra_driver.hpp"

using namespace dra;

static int failures = 0;
#define EXPECT_EQ(got, want) do { const std::string g_ = (got), w_ = (want); \
    if (g_ != w_) { printf("FAIL %s:%d\n  got:  %s\n  want: %s\n", __FILE__, __LINE__, g_.c_str(), w_.c_str()); ++failures; } } while (0)

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

static ClaimAllocation mig(const std::string& uid, const std::string& profile) {
    ClaimAllocation c; c.ClaimUID = uid; c.IsMig = true; c.Mig.Profile = profile; return c;
}
static ClaimAllocation gpu(const std::string& uid, uint32_t count = 1) {
    ClaimAllocation c; c.ClaimUID = uid; c.Gpu.Count = count; return c;
}

static std::string result(const ClaimAllocation& c) {
    std::string s = c.ClaimUID + " node=" + c.AllocatedNode + " error=" + c.Error;
    for (const auto& d : c.Allocation)
        s += " [" + d.Device + " " + std::to_string(d.GpuIndex) + " " + std::to_string(d.Start) + "+" + std::to_string(d.Size) +
             " " + std::to_string(d.GiProfileId) + "]";
    return s;
}

static Driver* make() {
    Driver* d = new Driver(0);
    d->SetMigProfiles(0, a100());
    d->SetNodes({node("node-a", 1, 0), node("node-b", 1, 0), node("node-c", 0, 2)});
    return d;
}

int main() {
    for (bool exhaustive : {false, true}) {
        // the claims of one batch, twice: one set for each Driver
        std::vector<ClaimAllocation> c[2];
        for (auto& v : c) v = {mig("c0", "3g.20gb"), mig("c1", "3g.20gb"), mig("c2", "3g.20gb"), mig("c3", "3g.20gb"),
                               gpu("w", 2), mig("bad", "9g.99gb")};
        auto pods = [&](std::vector<ClaimAllocation>& v) {
            std::vector<Driver::PodRequest> p(6);
            for (int i = 0; i < 4; ++i) { p[i].Claims = {&v[i]}; p[i].PotentialNodes = {"node-a"}; }
            p[3].PotentialNodes = {"node-a", "node-x", "node-b", "node-a"};
            p[4].Claims = {&v[4]}; p[4].PotentialNodes = {"node-a", "node-c"};
            p[5].Claims = {&v[5]}; p[5].PotentialNodes = {"node-a", "node-b"};
            return p;
        };
        Driver* d = make();
        Driver* ref = make();
        d->SetExhaustive(exhaustive); ref->SetExhaustive(exhaustive);
        // on the snapshot, every 3g pod sees node-a's two free slots
        EXPECT_EQ(d->UnsuitableReasonsBatch(pods(c[0]))[2], "1/1 nodes are available.");
        auto m = d->PlaceBatchWithReasons(pods(c[0]));
        ref->PlaceBatch(pods(c[1]));
        if (m.size() != 6) { printf("FAIL: %zu messages\n", m.size()); return 1; }
        EXPECT_EQ(m[0], "1/1 nodes are available.");
        EXPECT_EQ(m[1], "1/1 nodes are available.");
        // c0 and c1 took node-a's two 3g slots: the pod after them finds none
        EXPECT_EQ(m[2], "0/1 nodes are available: 1 node: claim \"c2\" (MIG 3g.20gb) no capacity.");
        // placed on node-b; node-a listed again after it is judged as the pod met it
        EXPECT_EQ(m[3], "1/4 nodes are available: 2 nodes: claim \"c3\" (MIG 3g.20gb) no capacity; 1 node: not in the inventory.");
        EXPECT_EQ(m[4], "1/2 nodes are available: 1 node: claim \"w\" (2 GPUs) no capacity.");
        EXPECT_EQ(m[5], "0/2 nodes are available: 2 nodes: claim \"bad\" (MIG 9g.99gb) unknown MIG profile '9g.99gb'.");
        for (size_t i = 0; i < c[0].size(); ++i) EXPECT_EQ(result(c[0][i]), result(c[1][i]));
        EXPECT_EQ(c[0][2].AllocatedNode, "");
        EXPECT_EQ(c[0][3].AllocatedNode, "node-b");
        EXPECT_EQ(c[0][4].AllocatedNode, "node-c");
        delete d; delete ref;
    }
    if (failures) { printf("place_why_test: %d failure(s)\n", failures); return 1; }
    printf("place_why_test ok\n");
    return 0;
}
