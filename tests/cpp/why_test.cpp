// why_test.cpp — exercises Driver::UnsuitableReasonsBatch of the C++ host layer (include/dra_driver.hpp): one
// kube-scheduler-style message per pod, naming the claim that blocks each group of nodes.  Needs an H100.
// Built by k8s-dra-driver_b200/build.py into tests/cpp/why_test; run by tests/test_gpu_unsuitable_why.py.
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

    auto w = gpu("w", 2), bad = mig("bad", "9g.99gb"), g3 = mig("g3", "3g.20gb");
    // t0 and t1 share a parent GPU: the lowering makes them adjacent, so the records are t0, t1, g1 — the blocking
    // claim g1 is record 2 while pod.Claims[2] is t1
    auto t0 = mig("t0", "1g.5gb", "shared"), g1 = gpu("g1", 1), t1 = mig("t1", "3g.20gb", "shared");
    Driver::PodRequest pw, pq, pb, pg;
    pw.Claims = {&w}; pw.PotentialNodes = {"node-a", "node-b", "node-c", "node-x"};
    pq.Claims = {&t0, &g1, &t1}; pq.PotentialNodes = {"node-a", "node-c"};
    pb.Claims = {&bad}; pb.PotentialNodes = {"node-a", "node-b"};
    pg.Claims = {&g3}; pg.PotentialNodes = {"node-b", "node-a"};
    for (bool exhaustive : {false, true}) {
        d.SetExhaustive(exhaustive);
        auto m = d.UnsuitableReasonsBatch({pw, pq, pb, pg});
        if (m.size() != 4) { printf("FAIL: %zu messages\n", m.size()); return 1; }
        EXPECT_EQ(m[0], "1/4 nodes are available: 2 nodes: claim \"w\" (2 GPUs) no capacity; 1 node: not in the inventory.");
        // node-a: the run {t0, t1} fits its one MIG GPU, g1 finds no full GPU.  node-c has no MIG GPU: in order, the run
        // fails as a run (its first member); with the search, g1 fits first and the pre-check finds no GPU offering 1g
        EXPECT_EQ(m[1], exhaustive
            ? "0/2 nodes are available: 1 node: claim \"g1\" (1 GPU) no capacity; 1 node: claim \"t0\" (MIG 1g.5gb) no GPU offers the MIG profile."
            : "0/2 nodes are available: 1 node: claim \"g1\" (1 GPU) no capacity; 1 node: claim \"t0\" (MIG 1g.5gb) co-located MIG devices do not fit on one parent GPU.");
        EXPECT_EQ(m[2], "0/2 nodes are available: 2 nodes: claim \"bad\" (MIG 9g.99gb) unknown MIG profile '9g.99gb'.");
        EXPECT_EQ(m[3], "2/2 nodes are available.");
    }
    // the message follows the inventory: after two 3g claims node-a is full for a third
    auto a = mig("a", "3g.20gb"), b = mig("b", "3g.20gb");
    d.Allocate({&a}, "node-a");
    d.Allocate({&b}, "node-a");
    d.SetExhaustive(false);
    EXPECT_EQ(d.UnsuitableReasonsBatch({pg})[0], "1/2 nodes are available: 1 node: claim \"g3\" (MIG 3g.20gb) no capacity.");

    if (failures) { printf("why_test: %d failure(s)\n", failures); return 1; }
    printf("why_test ok\n");
    return 0;
}
