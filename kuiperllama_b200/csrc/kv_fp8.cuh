// The fp8 KV cache's element (KLLM_KV_FP8, DESIGN.md 5.12): an e4m3 code per cached element, with a static
// scale s per (layer, KV head).  Shared by the persistent engine's writers and readers (megakernel.cu) and the
// batched prefill's (prefill.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace kllm {

// The code of x at the scale whose fp32 inverse is inv: fp32(x * inv) rounded to nearest even and saturated to
// +-448 (cvt.rn.satfinite.e4m3x2.f32)
__device__ __forceinline__ uint8_t e4m3_encode(float x, float inv) {
  return static_cast<uint8_t>(__nv_cvt_float_to_fp8(__fmul_rn(x, inv), __NV_SATFINITE, __NV_E4M3));
}

// value(code), exact: e4m3 widens to f16 exactly (cvt.rn.f16x2.e4m3x2), and f16 to fp32
__device__ __forceinline__ float e4m3_value(uint8_t code) {
  const __half_raw h = __nv_cvt_fp8_to_halfraw(code, __NV_E4M3);
  return __half2float(__half(h));
}

// the values of the four codes of a 32-bit word, byte 0 in .x
__device__ __forceinline__ float4 e4m3x4_values(uint32_t w) {
  const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w & 0xffffu), __NV_E4M3);
  const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w >> 16), __NV_E4M3);
  const float2 a = __half22float2(__half2(lo)), b = __half22float2(__half2(hi));
  return make_float4(a.x, a.y, b.x, b.y);
}

}  // namespace kllm
