// How many clusters of 1 / 2 / 4 / 8 CTAs with the scan kernel's footprint (448 threads, ~222 KB of dynamic shared
// memory: one CTA per SM) can be resident at once?  A persistent kernel whose CTAs of a cluster share one token
// range needs ALL its clusters resident together, so this bounds the cluster sizes the scan kernel could use.
//   nvcc -gencode arch=compute_90a,code=sm_90a -o cluster_occupancy cluster_occupancy.cu && ./cluster_occupancy
#include <cstdio>
#include <cuda_runtime.h>

__global__ void __launch_bounds__(448, 1) footprint_kernel(int* out) {
  extern __shared__ char smem[];
  if (out && threadIdx.x == 0) out[blockIdx.x] = smem[0];
}

int main() {
  const int smem_bytes = 222 * 1024;
  cudaFuncSetAttribute(footprint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  cudaFuncSetAttribute(footprint_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s: %d SMs\n", prop.name, prop.multiProcessorCount);
  for (int cs : {1, 2, 4, 8, 16}) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(prop.multiProcessorCount / cs * cs);
    cfg.blockDim = dim3(448);
    cfg.dynamicSmemBytes = smem_bytes;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = -1;
    cudaError_t e = cudaOccupancyMaxActiveClusters(&n, footprint_kernel, &cfg);
    printf("cluster size %2d: max active clusters %3d (= %3d CTAs of %d SMs)%s%s\n", cs, n, n * cs,
           prop.multiProcessorCount, e == cudaSuccess ? "" : "  error: ", e == cudaSuccess ? "" : cudaGetErrorString(e));
  }
  return 0;
}
