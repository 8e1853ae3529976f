// Shared host/device helpers for libprl.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/prl.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libprl is written for sm_90a only"
#endif

namespace prl {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define PRL_CHECK_ARG(cond, ...)            \
  do {                                      \
    if (!(cond)) {                          \
      prl::set_error(__VA_ARGS__);          \
      return PRL_ERR_INVALID;               \
    }                                       \
  } while (0)

#define PRL_CUDA(expr)                                                            \
  do {                                                                            \
    cudaError_t _e = (expr);                                                      \
    if (_e != cudaSuccess) {                                                      \
      prl::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,               \
                     cudaGetErrorString(_e));                                     \
      return PRL_ERR_CUDA;                                                        \
    }                                                                             \
  } while (0)

#define PRL_LAUNCH_CHECK()                                                        \
  do {                                                                            \
    prl::count_launch();                                                          \
    cudaError_t _e = cudaGetLastError();                                          \
    if (_e != cudaSuccess) {                                                      \
      prl::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__,           \
                     cudaGetErrorString(_e));                                     \
      return PRL_ERR_CUDA;                                                        \
    }                                                                             \
  } while (0)

int num_sms();  // SM count of the current device (cached per device)
bool use_pdl();  // programmatic dependent launch for the token-step kernels (PRL_PDL=0 disables)

// Launch with the programmatic-stream-serialization attribute: the kernel may start while its
// predecessor on the stream is still draining; it must execute pdl_wait() before touching anything
// the predecessor wrote (or still reads).  Works under stream capture (programmatic graph edges).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = use_pdl() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE function attribute: remember the largest size granted
// on each device (one static SmemAttr per launch site) instead of a per-process flag.
constexpr int kMaxDevices = 16;
struct SmemAttr { int bytes[kMaxDevices]; };
template <typename K>
inline cudaError_t ensure_smem(K kernel, int smem, SmemAttr& st) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDevices) return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (st.bytes[dev] < smem) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    st.bytes[dev] = smem;
  }
  return cudaSuccess;
}

constexpr int kWarp = 32;

// PDL device side: let the next kernel of the stream start its prologue / weight prefetch now ...
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// ... and block until every prerequisite grid has completed and its writes are visible.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// streaming 128-bit loads/stores that do not pollute L1
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld_stream_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ld_stream_u2(const uint2* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
               : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream_u4(uint4* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream_u2(uint2* p, uint2 v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};"
               :: "l"(p), "r"(v.x), "r"(v.y) : "memory");
}

__device__ __forceinline__ float bf16_bits_to_float(uint32_t hi16) {
  return __uint_as_float(hi16 << 16);
}
// round-to-nearest-even fp32 -> bf16 bits (NaN preserved as quiet NaN)
__device__ __forceinline__ uint32_t float_to_bf16_bits(float f) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(f));
}

// counter-based RNG for Gumbel-max sampling: noise depends only on (seed, step, row, vocab id), so the fused
// head epilogue (gemm_tc.cu) and the stand-alone sampler (decode_ops.cu) draw identical samples
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ float gumbel(uint64_t seed, uint32_t step, uint32_t b, uint32_t v) {
  uint32_t x = mix32((uint32_t)seed ^ (v * 0x9E3779B9u));
  x = mix32(x ^ (uint32_t)(seed >> 32) ^ (step * 0x85EBCA6Bu) ^ (b * 0xC2B2AE35u));
  const float u = ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
  return -__logf(-__logf(u));
}


}  // namespace prl
