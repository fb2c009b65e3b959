// driver_test.cpp — exercises the C++ host layer (include/dra_driver.hpp) the way a Go table test would
// exercise controller.Driver: the in-tree quickstart shapes, names, per-claim errors.  Needs an H100.
// Built by k8s-dra-driver_b200/build.py into tests/cpp/driver_test; run by tests/test_gpu_driver_cpp.py.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "dra_driver.hpp"

using namespace dra;

static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); ++failures; } } while (0)
#define EXPECT_EQ_S(a, b) do { std::string a_ = (a), b_ = (b); if (a_ != b_) { printf("FAIL %s:%d  %s == %s  ('%s' vs '%s')\n", __FILE__, __LINE__, #a, #b, a_.c_str(), b_.c_str()); ++failures; } } while (0)

// synthetic A100-40GB table (spec appendix); ids 19/14/9/5/0 are the A100's NVML GI profile ids
static std::vector<MigProfileInfo> a100() {
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
static ClaimAllocation gpu(const std::string& uid, uint32_t count = 1, SharingStrategy s = SharingStrategy::None, int64_t limit = 0) {
    ClaimAllocation c; c.ClaimUID = uid; c.Gpu.Count = count; c.Gpu.Sharing.Strategy = s; c.Gpu.Sharing.MpsPinnedDeviceMemoryLimitBytes = limit; return c;
}

int main() {
    Driver d(0);
    d.SetMigProfiles(0, a100());
    // mig-parted-config.yaml:8-16 "half-balanced": GPUs 0-3 MIG-enabled, 4-7 not
    d.SetNodes({node("node-a", 4, 4), node("node-b", 0, 2)});

    // --- gpu-test4.yaml:19-44: one claim, four MIG requests, matchAttribute parentUUID ---------------
    {
        auto a = mig("pod0-a", "1g.5gb", "shared"), b = mig("pod0-b", "1g.5gb", "shared"),
             c = mig("pod0-c", "2g.10gb", "shared"), e = mig("pod0-d", "3g.20gb", "shared");
        d.Allocate({&a, &b, &c, &e}, "node-a");
        EXPECT(a.Error.empty() && b.Error.empty() && c.Error.empty() && e.Error.empty());
        EXPECT_EQ_S(a.Allocation[0].Device, "gpu-0-mig-19-0-1");
        EXPECT_EQ_S(b.Allocation[0].Device, "gpu-0-mig-19-1-1");
        EXPECT_EQ_S(c.Allocation[0].Device, "gpu-0-mig-14-2-2");
        EXPECT_EQ_S(e.Allocation[0].Device, "gpu-0-mig-9-4-4");
        EXPECT(d.BusyMask("node-a", 0) == 0xFF);
        // gpu-test1..3: full GPUs come from the non-MIG half (nvlib.go:152)
        auto g1 = gpu("pod1-gpu"), g2 = gpu("pod2-gpus", 3);
        d.Allocate({&g1}, "node-a");
        d.Allocate({&g2}, "node-a");
        EXPECT_EQ_S(g1.Allocation[0].Device, "gpu-4");
        EXPECT(g2.Allocation.size() == 3);
        EXPECT_EQ_S(g2.Allocation[0].Device, "gpu-5");
        EXPECT_EQ_S(g2.Allocation[2].Device, "gpu-7");
        auto g3 = gpu("pod3-gpu");
        d.Allocate({&g3}, "node-a");
        EXPECT_EQ_S(g3.Error, "no capacity on the selected node");
        EXPECT(g3.Allocation.empty());
        // Deallocate gives the devices back; a second Deallocate is a no-op
        d.Deallocate(g2); d.Deallocate(g2);
        d.Allocate({&g3}, "node-a");
        EXPECT_EQ_S(g3.Allocation[0].Device, "gpu-5");
        d.Deallocate(a);
        EXPECT(d.BusyMask("node-a", 0) == 0xFE);
    }
    // --- per-claim errors are strings, never exceptions --------------------------------------------------
    {
        auto bad = mig("bad-profile", "9g.90gb");
        d.Allocate({&bad}, "node-a");
        EXPECT_EQ_S(bad.Error, "unknown MIG profile '9g.90gb'");
        auto nowhere = gpu("nowhere");
        d.Allocate({&nowhere}, "node-zzz");
        EXPECT_EQ_S(nowhere.Error, "unknown node 'node-zzz'");
        auto m = mig("mig-on-b", "1g.5gb");
        d.Allocate({&m}, "node-b");                       // node-b has no MIG-enabled GPU (nvlib.go:316-318)
        EXPECT_EQ_S(m.Error, "no GPU on the selected node offers the MIG profile");
    }
    // --- MPS sharing with a pinned-memory limit (sharing.go:234-237 arithmetic; gpu-test5.yaml:45: 10Gi) --
    {
        auto s1 = gpu("mps-1", 1, SharingStrategy::MPS, 30ll << 30), s2 = gpu("mps-2", 1, SharingStrategy::MPS, 20ll << 30),
             ts = gpu("ts-1", 1, SharingStrategy::TimeSlicing), low = gpu("mps-low", 1, SharingStrategy::MPS, 1000000);
        d.Allocate({&s1}, "node-b"); d.Allocate({&s2}, "node-b"); d.Allocate({&ts}, "node-b"); d.Allocate({&low}, "node-b");
        EXPECT_EQ_S(s1.Allocation[0].Device, "gpu-0");
        EXPECT_EQ_S(s2.Allocation[0].Device, "gpu-1");    // 20 GiB no longer fit beside 30 GiB on a 40 GiB GPU
        EXPECT_EQ_S(ts.Allocation[0].Device, "gpu-0");
        EXPECT_EQ_S(low.Error, "invalid limit: value set too low");      // "1M" -> 0M, sharing_test.go "too low"
        uint32_t mib = 0;
        EXPECT(MegabyteMiB(1000000000ll, &mib) && mib == 953);           // sharing_test.go "unit conversion G to M"
        EXPECT(MegabyteMiB(10000000ll, &mib) && mib == 9);               // "unit conversion M to M"
    }
    // --- UnsuitableNodes: all-or-nothing per pod, the node goes to every claim's list ---------------------
    {
        d.SetNodes({node("n0", 1, 0), node("n1", 2, 0), node("n2", 0, 1)});
        auto a = mig("p-a", "3g.20gb", "g"), b = mig("p-b", "3g.20gb", "g"), c = mig("p-c", "7g.40gb");
        d.UnsuitableNodes({&a, &b, &c}, {"n0", "n1", "n2", "n-unknown"});
        // n0: one GPU cannot hold 2x3g + 7g; n1: gpu0 takes both 3g, gpu1 the 7g; n2: no MIG
        EXPECT(a.UnsuitableNodes.size() == 3 && b.UnsuitableNodes.size() == 3 && c.UnsuitableNodes.size() == 3);
        EXPECT_EQ_S(a.UnsuitableNodes[0], "n0"); EXPECT_EQ_S(a.UnsuitableNodes[1], "n2"); EXPECT_EQ_S(a.UnsuitableNodes[2], "n-unknown");
        EXPECT(d.BusyMask("n1", 0) == 0);                 // pure
        d.Allocate({&a, &b, &c}, "n1");
        EXPECT_EQ_S(a.Allocation[0].Device, "gpu-0-mig-9-0-4");
        EXPECT_EQ_S(b.Allocation[0].Device, "gpu-0-mig-9-4-4");
        EXPECT_EQ_S(c.Allocation[0].Device, "gpu-1-mig-0-0-8");
    }
    // --- spec §12: the exhaustive placement search behind the same surface (SetExhaustive) -----------------
    // VERDICT r01's counter-example: slice 4 of the only GPU is busy; {1g, 3g} in that order defeats in-order first-fit
    {
        NodeAllocationState n; n.Node = "frag";
        AllocatableGpu g; g.Index = 0; g.MigEnabled = true; g.MemoryBytes = 40ull << 30;
        g.MigDevices.push_back({"1g.5gb", {4, 1}});
        n.Gpus.push_back(g);
        d.SetNodes({n});
        auto a = mig("x-a", "1g.5gb"), b = mig("x-b", "3g.20gb");
        d.UnsuitableNodes({&a, &b}, {"frag"});
        EXPECT(a.UnsuitableNodes.size() == 1);            // default mode: a false negative
        a.UnsuitableNodes.clear(); b.UnsuitableNodes.clear();
        d.SetExhaustive(true);
        d.UnsuitableNodes({&a, &b}, {"frag"});
        EXPECT(a.UnsuitableNodes.empty() && b.UnsuitableNodes.empty());
        d.Allocate({&a, &b}, "frag");
        EXPECT(a.Error.empty() && b.Error.empty());
        EXPECT_EQ_S(a.Allocation[0].Device, "gpu-0-mig-19-5-1");
        EXPECT_EQ_S(b.Allocation[0].Device, "gpu-0-mig-9-0-4");
        // a pod that cannot fit takes nothing (atomic) and says so
        auto c = mig("x-c", "7g.40gb"), e = mig("x-d", "1g.5gb");
        d.Allocate({&e, &c}, "frag");
        EXPECT_EQ_S(c.Error, "the pod's claims do not fit on the selected node together");
        EXPECT_EQ_S(e.Error, "the pod's claims do not fit on the selected node together");
        EXPECT(d.BusyMask("frag", 0) == (0x10 | 0x20 | 0x0F));
        // group members separated by another claim still share a parent (made adjacent by the host layer)
        d.SetExhaustive(false);
        d.SetNodes({node("n0", 2, 2)});
        auto m1 = mig("s-1", "3g.20gb", "same"), gg = gpu("s-g"), m2 = mig("s-2", "3g.20gb", "same");
        d.Allocate({&m1, &gg, &m2}, "n0");
        EXPECT(m1.Error.empty() && gg.Error.empty() && m2.Error.empty());
        EXPECT(m1.Allocation[0].GpuIndex == m2.Allocation[0].GpuIndex);
    }
    // --- a shared claim of Count copies that fails part way gives back the copies it took -----------------------------
    // Two 40 GiB GPUs and a 30 GiB MPS limit: each GPU holds one copy.  Count = 3 takes gpu-0 and gpu-1, the third copy
    // finds no memory, and the claim fails as a whole.  Driver exposes no memory or share counts, so the rollback shows in
    // what can be allocated next: two Count = 1 claims land on gpu-0 and gpu-1, as on a fresh node.
    for (const bool exhaustive : {false, true}) {
        d.SetExhaustive(exhaustive);
        d.SetNodes({node("mps", 0, 2)});
        auto three = gpu("mps-3", 3, SharingStrategy::MPS, 30ll << 30);
        d.Allocate({&three}, "mps");
        // exhaustive: the pod fails as a whole on the device and nothing is taken, so the rollback releases nothing
        EXPECT_EQ_S(three.Error, exhaustive ? "the pod's claims do not fit on the selected node together"
                                            : "no shareable GPU with enough free memory");
        EXPECT(three.Allocation.empty() && three.AllocatedNode.empty());
        d.Deallocate(three);                              // never held: a no-op
        auto a = gpu("mps-a", 1, SharingStrategy::MPS, 30ll << 30), b = gpu("mps-b", 1, SharingStrategy::MPS, 30ll << 30),
             c = gpu("mps-c", 1, SharingStrategy::MPS, 30ll << 30);
        d.Allocate({&a}, "mps"); d.Allocate({&b}, "mps"); d.Allocate({&c}, "mps");
        EXPECT(a.Error.empty() && b.Error.empty() && a.Allocation.size() == 1 && b.Allocation.size() == 1);
        if (a.Allocation.size() == 1 && b.Allocation.size() == 1) {
            EXPECT_EQ_S(a.Allocation[0].Device, "gpu-0");
            EXPECT_EQ_S(b.Allocation[0].Device, "gpu-1");
        }
        EXPECT(!c.Error.empty() && c.Allocation.empty());  // and the node is full again, with no copy left over
        // released and taken again: the copies a Deallocate gives back are the copies a later claim gets
        d.Deallocate(b);
        auto e = gpu("mps-e", 1, SharingStrategy::MPS, 30ll << 30);
        d.Allocate({&e}, "mps");
        EXPECT(e.Allocation.size() == 1 && e.Allocation[0].Device == "gpu-1");
    }
    d.SetExhaustive(false);
    if (failures) { printf("%d FAILED\n", failures); return 1; }
    printf("driver_test: all checks passed\n");
    return 0;
}
