// Developer probe: how many clusters of 2 / 4 / 8 CTAs with ~226 KB of dynamic shared memory (one CTA per SM) are co-resident?
// nvcc -gencode arch=compute_90a,code=sm_90a -o /tmp/cluster_occ tools/probes/cluster_occ.cu
#include <cuda_runtime.h>
#include <cstdio>
__global__ void dummy(int* p) { extern __shared__ char s[]; if (p) p[0] = s[0]; }
int main() {
  const int smem = 226 * 1024;
  cudaFuncSetAttribute(dummy, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(dummy, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  for (int cs : {1, 2, 4, 8, 16}) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(132 / cs * cs); cfg.blockDim = dim3(320); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute a[1];
    a[0].id = cudaLaunchAttributeClusterDimension; a[0].val.clusterDim.x = cs; a[0].val.clusterDim.y = 1; a[0].val.clusterDim.z = 1;
    cfg.attrs = a; cfg.numAttrs = 1;
    int n = -1;
    cudaError_t e = cudaOccupancyMaxActiveClusters(&n, dummy, &cfg);
    printf("cluster %2d: max active clusters %d (%d SMs) %s\n", cs, n, n * cs, e == cudaSuccess ? "" : cudaGetErrorString(e));
  }
  return 0;
}
