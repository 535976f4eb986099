// rt_occupancy.cu — how many clusters of k_rt_group<M> an H100 keeps resident (cudaOccupancyMaxActiveClusters) at
// cluster sizes 2, 4, 8 and 16, for M = 128 and 512.  Built and run by tools/group_bench.py --occupancy.
#include <cstdio>

#include <cuda_runtime.h>

#include "../reevr_b200/csrc/kernels_rt.cuh"

template <int M>
static void report(int C) {
  const int smem = pc::rt_smem_layout(M, C).bytes;
  cudaFuncSetAttribute(pc::k_rt_group<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, pc::rt_smem_layout(M, 16).bytes);
  cudaFuncSetAttribute(pc::k_rt_group<M>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  for (int cs = 2; cs <= 16; cs *= 2) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cs * 32, 1, 1);
    cfg.blockDim = dim3(256, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = -1;
    const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, pc::k_rt_group<M>, &cfg);
    std::printf("{\"M\": %d, \"C\": %d, \"smem\": %d, \"cluster\": %d, \"max_active_clusters\": %d, \"err\": \"%s\"}\n", M,
                C, smem, cs, n, cudaGetErrorString(e));
  }
}

int main() {
  report<128>(4);
  report<512>(4);
  return 0;
}
