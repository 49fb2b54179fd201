// Shared helpers for the rnc kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>
#include "rnc.h"

namespace rnc {

extern thread_local int g_last_cuda_error;
extern thread_local long long g_launch_count;

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
__device__ __forceinline__ bool aligned16_dev(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

#define RNC_XSTR(x) #x
#define RNC_STR(x) RNC_XSTR(x)
#define RNC_STR_CUDA RNC_STR(__CUDACC_VER_MAJOR__) "." RNC_STR(__CUDACC_VER_MINOR__)

// Opt a kernel into > 48 KB of dynamic shared memory, once per device.
template <typename K>
inline int ensure_dyn_smem(K kernel, int bytes, unsigned long long* done_mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (__atomic_load_n(done_mask, __ATOMIC_ACQUIRE) & bit) return RNC_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) { g_last_cuda_error = static_cast<int>(e); return RNC_ERR_CUDA; }
  __atomic_fetch_or(done_mask, bit, __ATOMIC_RELEASE);
  return RNC_OK;
}

// Record a launch and translate the launch status.
inline int after_launch(int n = 1) {
  g_launch_count += n;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    g_last_cuda_error = static_cast<int>(e);
    return RNC_ERR_CUDA;
  }
  return RNC_OK;
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Carves a workspace into buffers, in the order take() is called, each starting on a 16-byte boundary.  On a null base it
// only counts: a layout function run once on nullptr gives the workspace's size in `bytes` and run on the real base gives its
// pointers, so the two cannot disagree.
struct Carve {
  char* base;
  size_t bytes = 0;
  template <typename T>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += (n * sizeof(T) + 15) & ~size_t(15);
    return p;
  }
};

// Programmatic dependent launch (PDL).  A kernel launched with launch_pdl() may start while its predecessor in the stream is
// still draining: it runs its prologue (barrier init, descriptor prefetch), then pdl_wait() blocks until the
// predecessor has completed and its writes are visible.  pdl_trigger() in the predecessor lets the dependent start early;
// without it the dependent starts at the predecessor's exit (plain stream order).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Exact hi/lo split of a pair of floats into halves: hi = rn(v) saturated to +-65504 (one F2FP.SATFINITE), lo = rn(v - hi).
// |v| <= 65504: hi + lo reproduces v to 22 significant bits.  Beyond the half range both parts saturate (finite, never inf).
__device__ __forceinline__ uint32_t pack_half2_sat(float lo_elem, float hi_elem) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
  return r;
}
__device__ __forceinline__ void split_pair(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  hi = pack_half2_sat(v0, v1);
  const float2 back = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = pack_half2_sat(v0 - back.x, v1 - back.y);
}

// Two independent fp32 FMAs on a pair of adjacent outputs (Hopper has no packed fp32 FMA; each lane rounds as fmaf does).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// Gate activations of the tensor-core epilogues: ex2.approx / rcp.approx based, a few instructions, branch-free (the libm
// forms cost 30-40 instructions each and the GRU epilogues are latency-bound on them).  Measured over every 22-bit-significand
// input of 2^-24 .. 2^8 on an H100 SXM (tests/test_gpu_conv_epilogue_model.py): sigmoid_fast's relative error is at most
// 1.82e-7 + 1.06e-7 |x| (exp's argument rounding grows with |x|; 3.9e-6 at |x| = 128), and it returns 0 for x <= -87.34
// (rcp.approx.ftz flushes results below 2^-126); tanh_fast's is at most 4.3e-7 (just above the 0.25 branch), 8.9e-8 on the
// Taylor branch.
__device__ __forceinline__ float fast_rcp(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sigmoid_fast(float x) {
  return fast_rcp(1.0f + __expf(-x));                    // x << 0: exp -> inf, rcp -> 0; x >> 0: -> 1
}
__device__ __forceinline__ float tanh_fast(float x) {
  const float ax = fabsf(x), x2 = x * x;
  // |x| < 0.25: odd Taylor series through x^9 (truncation < 1e-8 relative); otherwise 1 - 2 / (exp(2|x|) + 1)
  const float poly = x * (1.0f + x2 * (-0.33333334f + x2 * (0.13333334f + x2 * (-0.05396825f + x2 * 0.021869488f))));
  const float big = 1.0f - 2.0f * fast_rcp(__expf(2.0f * fminf(ax, 20.0f)) + 1.0f);
  return ax < 0.25f ? poly : copysignf(big, x);
}

}  // namespace rnc
