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

// ---- programmatic dependent launch (PDL), opt-in with RSTNET_PDL=1.  The LM frame is a chain of ~800 small dependent
// kernels; with the launch attribute below the next kernel's CTAs are scheduled while the previous grid drains and run their
// prologue (barrier set-up, descriptor prefetch) up to `pdl_wait()`, which returns once the previous grid has
// completed and flushed.  Every kernel launched through launch_pdl() calls pdl_launch_dependents() and then pdl_wait()
// before its first global access, so the ordering guarantees are those of plain stream order (also inside a captured CUDA
// graph).  Off by default: inside a replayed CUDA graph, programmatic edges between kernel nodes can cost more per launch
// than plain edges, which outweighs the hidden prologues (time the frame with scripts/lm_frame_timing.py before enabling
// it).  Without the attribute griddepcontrol.* are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_enabled();   // env RSTNET_PDL=1 (default off); capi.cu

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
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
