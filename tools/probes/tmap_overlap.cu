// Developer probe: does cuTensorMapEncodeTiled accept a sliding-window (overlapping) view — stride of dimension 1 (16 B)
// smaller than the extent of dimension 0 (128 B) — and does the TMA unit load it as expected?
// nvcc -gencode arch=compute_90a,code=sm_90a -o /tmp/tmap_overlap tools/probes/tmap_overlap.cu -lcuda
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

__global__ void probe(const __grid_constant__ CUtensorMap m, unsigned short* out, int x0, int y0) {
  __shared__ __align__(1024) unsigned short tile[128 * 64];
  __shared__ uint64_t bar;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(&bar)), "r"(128 * 64 * 2));
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(tile)), "l"(&m), "r"((uint32_t)__cvta_generic_to_shared(&bar)),
                   "r"(0), "r"(x0), "r"(y0), "r"(0) : "memory");
  }
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"((uint32_t)__cvta_generic_to_shared(&bar)) : "memory");
  }
  for (int i = threadIdx.x; i < 128 * 64; i += blockDim.x) out[i] = tile[i];
}

int main() {
  const int pitch = 4128, rows = 16, OW = 512;             // halves per row; 1032 px x 4 ch
  std::vector<unsigned short> h(pitch * rows + 256);
  for (size_t i = 0; i < h.size(); ++i) h[i] = (unsigned short)(i % 60000);
  unsigned short *d, *o;
  cudaMalloc(&d, h.size() * 2); cudaMalloc(&o, 128 * 64 * 2);
  cudaMemcpy(d, h.data(), h.size() * 2, cudaMemcpyHostToDevice);
  CUtensorMap m;
  const cuuint64_t dims[4] = {64, (cuuint64_t)OW, (cuuint64_t)rows, 1};
  const cuuint64_t strides[3] = {16, (cuuint64_t)pitch * 2, (cuuint64_t)pitch * 2 * rows};
  const cuuint32_t box[4] = {64, 128, 2, 1};
  const cuuint32_t es[4] = {1, 1, 2, 1};
  CUresult r = cuTensorMapEncodeTiled(&m, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, d, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  printf("encode overlapping 4-D view: %d\n", (int)r);
  if (r != CUDA_SUCCESS) return 1;
  const int x0 = 128, y0 = 3;
  probe<<<1, 128>>>(m, o, x0, y0);
  cudaError_t e = cudaDeviceSynchronize();
  printf("kernel: %s\n", cudaGetErrorString(e));
  std::vector<unsigned short> res(128 * 64);
  cudaMemcpy(res.data(), o, res.size() * 2, cudaMemcpyDeviceToHost);
  int bad = 0;
  for (int r_ = 0; r_ < 128; ++r_)
    for (int e_ = 0; e_ < 64; ++e_) {
      const size_t src = (size_t)y0 * pitch + (size_t)(x0 + r_) * 8 + e_;
      if (res[r_ * 64 + e_] != (unsigned short)(src % 60000)) ++bad;
    }
  printf("mismatches: %d of %d\n", bad, 128 * 64);
  // negative start row -> zero fill
  probe<<<1, 128>>>(m, o, 0, -1);
  cudaDeviceSynchronize();
  cudaMemcpy(res.data(), o, res.size() * 2, cudaMemcpyDeviceToHost);
  int nz = 0;
  for (auto v : res) nz += v != 0;
  printf("row -1: nonzero %d (expect 0)\n", nz);
  return bad != 0;
}
