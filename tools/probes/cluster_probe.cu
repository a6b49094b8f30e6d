// How many clusters of size S (512 threads, 128 KB smem per CTA: the k_jacobi<512> footprint) are co-resident
// on this GPU, and where do they land?   nvcc -gencode arch=compute_90a,code=sm_90a -o cluster_probe cluster_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <cooperative_groups.h>
namespace cg = cooperative_groups;
__global__ void spin(unsigned long long* start, unsigned* smid, unsigned long long ns) {
    extern __shared__ float sm[];
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    unsigned id;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(id));
    if (threadIdx.x == 0) { start[blockIdx.x] = t0; smid[blockIdx.x] = id; sm[0] = 1.f; }
    cg::this_cluster().sync();
    unsigned long long t;
    do { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); } while (t - t0 < ns);
    cg::this_cluster().sync();
}
int main() {
    const int smem = 64 * 512 * 4 + 64;
    cudaFuncSetAttribute(spin, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(spin, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    unsigned long long* start; unsigned* smid;
    cudaMallocManaged(&start, 4096 * 8); cudaMallocManaged(&smid, 4096 * 4);
    for (int S : {1, 2, 4, 8, 16}) {
      for (int pol = 0; pol < 3; ++pol) {
        const int nclusters = 40;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(S * nclusters); cfg.blockDim = dim3(512); cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[2];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = S; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        at[1].id = cudaLaunchAttributeClusterSchedulingPolicyPreference;
        at[1].val.clusterSchedulingPolicyPreference = pol == 1 ? cudaClusterSchedulingPolicySpread : pol == 2 ? cudaClusterSchedulingPolicyLoadBalancing : cudaClusterSchedulingPolicyDefault;
        cfg.attrs = at; cfg.numAttrs = 2;
        int maxc = -1;
        cudaError_t e = cudaOccupancyMaxActiveClusters(&maxc, spin, &cfg);
        e = cudaLaunchKernelEx(&cfg, spin, start, smid, 2000000ull);
        cudaError_t e2 = cudaDeviceSynchronize();
        if (e != cudaSuccess || e2 != cudaSuccess) { printf("S=%d pol=%d launch error %s %s\n", S, pol, cudaGetErrorString(e), cudaGetErrorString(e2)); continue; }
        unsigned long long t0 = ~0ull; for (int i = 0; i < S * nclusters; ++i) if (start[i] < t0) t0 = start[i];
        int first = 0; for (int c = 0; c < nclusters; ++c) if (start[c * S] - t0 < 1000000ull) ++first;
        printf("S=%2d policy=%d  occupancy API max clusters %3d ; measured first-wave clusters %3d (= %3d SMs)\n", S, pol, maxc, first, first * S);
        if (S == 8 && pol == 0) { for (int c = 0; c < first; ++c) { printf("  cluster %2d SMs:", c); for (int k = 0; k < S; ++k) printf(" %3u", smid[c * S + k]); printf("\n"); } }
      }
    }
    return 0;
}
