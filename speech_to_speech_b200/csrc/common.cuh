// common.cuh -- shared device/host helpers for libs2s_b200 (sm_90a, Hopper).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/s2s_b200.h"

// ------------------------------------------------------------------------------------------
// host-side error plumbing
// ------------------------------------------------------------------------------------------
void s2s_set_error(const char* fmt, ...);
void s2s_count_launch(int n = 1);

#define S2S_CHECK_CUDA(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      s2s_set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, cudaGetErrorName(_e),  \
                    cudaGetErrorString(_e));                                              \
      return S2S_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define S2S_CHECK(expr)        \
  do {                         \
    int _r = (expr);           \
    if (_r != S2S_OK) return _r; \
  } while (0)

#define S2S_REQUIRE(cond, ...)        \
  do {                                \
    if (!(cond)) {                    \
      s2s_set_error(__VA_ARGS__);     \
      return S2S_ERR_INVALID;         \
    }                                 \
  } while (0)

#define S2S_LAUNCH_CHECK()                 \
  do {                                     \
    s2s_count_launch();                    \
    S2S_CHECK_CUDA(cudaGetLastError());    \
  } while (0)

struct s2s_ctx {
  int device;
  int num_sms;
  // SM partition ("lane"): the persistent cooperative decode kernels launched through this context use this many CTAs
  // (0 = one per SM).  Two contexts of half the SMs each run their decode launches side by side on one GPU: the phases of a
  // decode step are latency-bound, so two half-grid launches finish in about the time of one whole-grid launch.
  int decode_ctas;
  // cuTensorMapEncodeTiled resolved through the runtime (no link-time libcuda dependency)
  void* encode_tiled;
};

// Opt a kernel in to the device's largest dynamic shared-memory size (227 KB minus its static shared memory) ONCE per process.
// The attribute is per function, not per launch: host threads of different lanes launch the same kernel with different
// sizes at the same time, and "set the size I need, then launch" races (a smaller size set by the other thread in between
// makes the launch fail with cudaErrorLaunchOutOfResources).  The maximum is valid for every launch.
template <typename K>
inline cudaError_t s2s_opt_in_max_smem(K kern, int device, size_t need, const char** why) {
  static thread_local const void* last_ok = nullptr;   // fast path: this thread already saw this kernel opted in
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, (const void*)kern);
  if (e != cudaSuccess) return e;
  int optin = 0;
  e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  if (e != cudaSuccess) return e;
  const long long max_dyn = (long long)optin - (long long)fa.sharedSizeBytes;
  if ((long long)need > max_dyn) { if (why) *why = "dynamic shared memory exceeds the device limit"; return cudaErrorInvalidValue; }
  if (last_ok == (const void*)kern && fa.maxDynamicSharedSizeBytes >= max_dyn) return cudaSuccess;
  e = cudaFuncSetAttribute((const void*)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_dyn);
  if (e == cudaSuccess) last_ok = (const void*)kern;
  return e;
}

inline int dec_grid(const s2s_ctx* c) { return (c->decode_ctas > 0 && c->decode_ctas < c->num_sms) ? c->decode_ctas : c->num_sms; }

// ------------------------------------------------------------------------------------------
// dtype helpers
// ------------------------------------------------------------------------------------------
template <typename T> struct DT;
template <> struct DT<__half> {
  static constexpr int code = S2S_F16;
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  __device__ __forceinline__ static float to_f(__half v) { return __half2float(v); }
  __device__ __forceinline__ static __half from_f(float v) { return __float2half_rn(v); }
  __device__ __forceinline__ static float2 to_f2(uint32_t u) {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
  __device__ __forceinline__ static uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};
template <> struct DT<__nv_bfloat16> {
  static constexpr int code = S2S_BF16;
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  __device__ __forceinline__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ __forceinline__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
  __device__ __forceinline__ static float2 to_f2(uint32_t u) {
    // bf16 -> f32 is a 16-bit shift
    float2 r;
    r.x = __uint_as_float(u << 16);
    r.y = __uint_as_float(u & 0xFFFF0000u);
    return r;
  }
  __device__ __forceinline__ static uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
};

// ------------------------------------------------------------------------------------------
// warp / math helpers
// ------------------------------------------------------------------------------------------
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
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// 16-byte read-only streaming load (weights are read once per step: do not pollute L1)
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ------------------------------------------------------------------------------------------
// mbarrier / TMA PTX wrappers (sm_90a)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (-> CUDA error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(desc) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(desc), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(desc), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
