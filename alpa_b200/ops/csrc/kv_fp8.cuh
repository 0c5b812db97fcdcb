// The fp8 KV-cache row format, shared by the decode, ragged and cache store / load kernels.
//
// One cache row of one (token, K/V head) holds D e4m3 values q and one fp32 scale s:
//   s = max(amax, 1e-8) / 448      amax = max |x| over the row's D bf16 values
//   q = e4m3_rne(x / s)            the value read back is float(q) * s
// Both divisions are correctly rounded (the library is built with --use_fast_math, where `/` is approximate), so the
// bytes equal PyTorch's `(x.float() / s).to(torch.float8_e4m3fn)`.  |x / s| <= 448 (up to the rounding of s, which
// rounds to 448), so the hardware's satfinite conversion and PyTorch's cast agree.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <stdint.h>

namespace ab {

__device__ __forceinline__ float kv_fp8_scale(float amax) { return __fdiv_rn(fmaxf(amax, 1e-8f), 448.f); }

// x[8] -> 8 e4m3 bytes (channel i in byte i)
__device__ __forceinline__ uint2 kv_fp8_quant8(const float* x, float s) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    w[i] = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(x[2 * i], s), __fdiv_rn(x[2 * i + 1], s)), __NV_SATFINITE,
                                    __NV_E4M3);
  return make_uint2(w[0] | (w[1] << 16), w[2] | (w[3] << 16));
}

// two e4m3 bytes (channel 0 in the low byte) -> their exact values
__device__ __forceinline__ float2 kv_fp8_unpack2(uint32_t two) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(two & 0xffffu), __NV_E4M3);
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}

// 8 e4m3 bytes -> f[8]
__device__ __forceinline__ void kv_fp8_unpack8(uint2 q, float* f) {
  float2 t;
  t = kv_fp8_unpack2(q.x); f[0] = t.x; f[1] = t.y;
  t = kv_fp8_unpack2(q.x >> 16); f[2] = t.x; f[3] = t.y;
  t = kv_fp8_unpack2(q.y); f[4] = t.x; f[5] = t.y;
  t = kv_fp8_unpack2(q.y >> 16); f[6] = t.x; f[7] = t.y;
}

// 8 bf16 channels (one 16-byte piece) -> f[8], and their largest magnitude
__device__ __forceinline__ float kv_bf16_unpack8(int4 v, float* f) {
  const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u[i]));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
    amax = fmaxf(amax, fmaxf(fabsf(t.x), fabsf(t.y)));
  }
  return amax;
}

}  // namespace ab
