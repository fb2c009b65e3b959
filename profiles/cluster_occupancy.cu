// cluster_occupancy.cu — how many thread-block clusters of CL CTAs fit on the device at once (profiles/, not product code).
//
// A cluster form of the single-launch Allocate kernel (DESIGN.md §8, 2c) runs one CTA of 8 warps per node with a
// 16-byte receive slot per claim (the cfg2 batch: 10,000 claims, ~160 KB), so one CTA per SM.  A cluster of CL CTAs
// must sit inside one GPC; SMs of a GPC that do not fill a whole cluster stay idle.  cudaOccupancyMaxActiveClusters
// answers for the device at hand; the grid must fit in that many clusters for the launch to stay in one wave.
//
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o cluster_occupancy cluster_occupancy.cu && ./cluster_occupancy [n_claim]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstdint>
#include <cuda_runtime.h>

__global__ void __launch_bounds__(256, 1) k_probe(int* p) {
    extern __shared__ int s[];
    if (p) p[threadIdx.x] = s[threadIdx.x];
}

int main(int argc, char** argv) {
    const unsigned n_claim = argc > 1 ? (unsigned)atoi(argv[1]) : 10000u;
    cudaDeviceProp pr;
    if (cudaGetDeviceProperties(&pr, 0) != cudaSuccess) { fprintf(stderr, "no CUDA device\n"); return 1; }
    // receive area (16 B per claim) + the fixed head of the layout (table, barriers, inventory, live list, counts)
    const size_t smem = 4096 + (size_t)n_claim * 16;
    cudaFuncSetAttribute(k_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int nb = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_probe, 256, smem);
    printf("%s, %d SMs, %zu B dynamic shared memory per CTA, %d CTA(s)/SM\n", pr.name, pr.multiProcessorCount, smem, nb);
    for (int cl = 2; cl <= 8; cl *= 2) {
        cudaLaunchConfig_t lc; memset(&lc, 0, sizeof lc);
        lc.gridDim = dim3(cl * 64); lc.blockDim = dim3(256); lc.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        lc.attrs = at; lc.numAttrs = 1;
        int ncl = 0;
        const cudaError_t e = cudaOccupancyMaxActiveClusters(&ncl, k_probe, &lc);
        printf("CL=%d: %d clusters at once = %d CTAs%s%s\n", cl, ncl, ncl * cl, e == cudaSuccess ? "" : "  error: ",
               e == cudaSuccess ? "" : cudaGetErrorString(e));
    }
    return 0;
}
