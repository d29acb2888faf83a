// Shared helpers for the sm_90a kernels of libar_b200.so.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ar_b200.h"

namespace ar {

void set_error(const char* fmt, ...);

#define AR_REQUIRE(cond, code, ...)      \
  do {                                   \
    if (!(cond)) {                       \
      ar::set_error(__VA_ARGS__);        \
      return (code);                     \
    }                                    \
  } while (0)

#define AR_CHECK_LAUNCH()                                              \
  do {                                                                 \
    cudaError_t e__ = cudaGetLastError();                              \
    if (e__ != cudaSuccess) {                                          \
      ar::set_error("%s:%d launch failed: %s", __FILE__, __LINE__,     \
                    cudaGetErrorString(e__));                          \
      return (int)e__;                                                 \
    }                                                                  \
  } while (0)

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

__device__ __forceinline__ float bf16_bits_to_f32(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }
__device__ __forceinline__ uint16_t f32_to_bf16_bits(float f) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}
__device__ __forceinline__ float f16_round(float f) { return __half2float(__float2half_rn(f)); }
__device__ __forceinline__ float bf16_round(float f) { return __bfloat162float(__float2bfloat16_rn(f)); }

// torch's float -> float8_e4m3fn (RNE, no saturation needed: callers clamp to +-448 first)
__device__ __forceinline__ uint8_t f32_to_e4m3_bits(float f) {
  return (uint8_t)__nv_cvt_float_to_fp8(f, __NV_SATFINITE, __NV_E4M3);
}
__device__ __forceinline__ float e4m3_bits_to_f32(uint8_t b) {
  __half_raw h = __nv_cvt_fp8_to_halfraw(b, __NV_E4M3);
  return __half2float(*reinterpret_cast<__half*>(&h));
}

struct alignas(16) U4 { uint32_t x, y, z, w; };
struct alignas(8) U2 { uint32_t x, y; };

int sm_count();

}  // namespace ar
