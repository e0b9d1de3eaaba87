// Shared helpers for the rstnet_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

namespace rstnet {

// thread-local last error text, exported through rstnet_last_error()
void set_error(const char* fmt, ...);
int  check_launch(const char* what);

#define RSTNET_REQUIRE(cond, ...)                      \
  do {                                                 \
    if (!(cond)) {                                     \
      ::rstnet::set_error(__VA_ARGS__);                \
      return 1;                                        \
    }                                                  \
  } while (0)

enum Act : int { ACT_NONE = 0, ACT_ELU = 1, ACT_GELU = 2 };

// ELU(alpha=1) exactly as ATen's CPU kernel evaluates it: x <= 0 ? exp(x) - 1 : x
// (aten/src/ATen/native/cpu/Activation.cpp elu_kernel; not expm1).
__device__ __forceinline__ float elu_f(float x) { return x <= 0.f ? (expf(x) - 1.0f) : x; }
// exact (erf) GELU, torch.nn.functional.gelu default
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_ELU) return elu_f(x);
  if (act == ACT_GELU) return gelu_f(x);
  return x;
}

// Tensor-core epilogues: ELU through ex2.approx (|abs error| ~2e-7, below the 3xTF32 product error of the GEMM that
// feeds it); the CUDA-core kernels keep expf.  The full-precision version cost more than the tile's MMAs.
__device__ __forceinline__ float elu_fast(float x) { return x > 0.f ? x : __expf(x) - 1.f; }
template <int ACTC>
__device__ __forceinline__ float4 apply_act4_tc(float4 v) {
  if (ACTC == ACT_ELU) return make_float4(elu_fast(v.x), elu_fast(v.y), elu_fast(v.z), elu_fast(v.w));
  if (ACTC == ACT_GELU) return make_float4(gelu_f(v.x), gelu_f(v.y), gelu_f(v.z), gelu_f(v.w));
  return v;
}

__device__ __forceinline__ float4 apply_act4_tc(float4 v, int act) {
  if (act == ACT_ELU) return apply_act4_tc<ACT_ELU>(v);
  if (act == ACT_GELU) return apply_act4_tc<ACT_GELU>(v);
  return v;
}

// four lanes of one activation with the selector tested once (keeps rolled epilogue loops small)
__device__ __forceinline__ float4 apply_act4(float4 v, int act) {
  if (act == ACT_ELU) return make_float4(elu_f(v.x), elu_f(v.y), elu_f(v.z), elu_f(v.w));
  if (act == ACT_GELU) return make_float4(gelu_f(v.x), gelu_f(v.y), gelu_f(v.z), gelu_f(v.w));
  return v;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, int src_bytes) {
  uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem_src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// SMs of the current device (grid sizing of persistent and grid-stride kernels)
inline int sm_count() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 1;
}

// One-time opt-in to more than 48 KB of dynamic shared memory.  The attribute belongs to the (function, device) pair, so
// the "done" mask is keyed by the CURRENT device ordinal: a second GPU in the same process gets its own opt-in.
template <typename Kernel>
inline void smem_optin(Kernel* kernel, int bytes, unsigned long long& done_mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(done_mask & bit)) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    done_mask |= bit;
  }
}

}  // namespace rstnet
