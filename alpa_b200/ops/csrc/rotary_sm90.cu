// Bandwidth-bound sm_90a kernels of the Llama-style block: rotary position embedding on the packed QKV tensor and the
// SwiGLU activation (forward and backward) on interleaved gate / up pairs.  bf16 in and out, fp32 math, one rounding.
#include "kernels.h"
#include "ptx.cuh"

namespace ab {

// ------------------------------------------------------------------------------------------------
// Rotary embedding.  x / y: [tokens, heads = Hkv * slots, D] with slots = G + 2; slots 0..G (the G query heads and K)
// rotate in HF's rotate_half convention (element i pairs with i + D/2 at angle float(pos) * inv_freq[i]), slot G + 1
// (V) is copied.  One CTA per token (grid-stride): cos / sin of the token's D/2 angles are computed once into shared
// memory and reused by every head; each thread then moves 8 elements of each half of one head per step.
// ------------------------------------------------------------------------------------------------
constexpr int kRopeThreads = 128;

__global__ void __launch_bounds__(kRopeThreads)
rotary_packed_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                     const int64_t* __restrict__ pos, const float* __restrict__ inv_freq, int tokens, int heads,
                     int slots, int D, int inverse) {
  extern __shared__ float2 cs[];  // [D / 2] (cos, +-sin) of this token
  const int half = D / 2, vph = half / 8;
  const int units = heads * vph;
  for (int t = blockIdx.x; t < tokens; t += gridDim.x) {
    const float p = (float)pos[t];
    __syncthreads();  // the previous token's readers of cs are done
    for (int i = threadIdx.x; i < half; i += blockDim.x) {
      const float ang = p * inv_freq[i];  // the fp32 product HF forms
      // Double precision: under --use_fast_math sincosf becomes MUFU.SIN / MUFU.COS without range reduction, which
      // is wrong at the thousands of radians ordinary positions reach.  One evaluation per (token, frequency).
      double s, c;
      sincos((double)ang, &s, &c);
      cs[i] = make_float2((float)c, inverse ? -(float)s : (float)s);
    }
    __syncthreads();
    const size_t base = (size_t)t * heads * D;
    for (int u = threadIdx.x; u < units; u += blockDim.x) {
      const int hp = u / vph, c0 = (u - hp * vph) * 8;
      const size_t off = base + (size_t)hp * D + c0;
      int4 a = ld_nc_v4(x + off), b = ld_nc_v4(x + off + half);
      if (hp % slots != slots - 1) {
        uint32_t* au = reinterpret_cast<uint32_t*>(&a);
        uint32_t* bu = reinterpret_cast<uint32_t*>(&b);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 x1 = unpack_bf16x2(au[j]), x2 = unpack_bf16x2(bu[j]);
          const float2 k0 = cs[c0 + 2 * j], k1 = cs[c0 + 2 * j + 1];
          au[j] = pack_bf16x2(x1.x * k0.x - x2.x * k0.y, x1.y * k1.x - x2.y * k1.y);
          bu[j] = pack_bf16x2(x2.x * k0.x + x1.x * k0.y, x2.y * k1.x + x1.y * k1.y);
        }
      }
      *reinterpret_cast<int4*>(y + off) = a;
      *reinterpret_cast<int4*>(y + off + half) = b;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// SwiGLU on gu [n, 2] (pair j = (gate j, up j)): h = silu(g) * u.  Backward recomputes from gu:
// dg = dh * u * s (1 + g (1 - s)), du = dh * silu(g), s = sigmoid(g).  4 pairs (16 bytes of gu) per thread per step.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float g) { return 1.f / (1.f + __expf(-g)); }

__global__ void __launch_bounds__(256)
swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ h, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const int4 v = ld_nc_v4(gu + i * 8);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      o[j] = f.x * sigmoidf_(f.x) * f.y;
    }
    *reinterpret_cast<uint2*>(h + i * 4) = make_uint2(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]));
  }
}

__global__ void __launch_bounds__(256)
swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ gu,
                  __nv_bfloat16* __restrict__ dgu, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    int4 v = ld_nc_v4(gu + i * 8);
    const uint2 d = *reinterpret_cast<const uint2*>(dh + i * 4);
    uint32_t* w = reinterpret_cast<uint32_t*>(&v);
    const float2 d01 = unpack_bf16x2(d.x), d23 = unpack_bf16x2(d.y);
    const float dv[4] = {d01.x, d01.y, d23.x, d23.y};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      const float s = sigmoidf_(f.x);
      w[j] = pack_bf16x2(dv[j] * f.y * s * (1.f + f.x * (1.f - s)), dv[j] * f.x * s);
    }
    *reinterpret_cast<int4*>(dgu + i * 8) = v;
  }
}

}  // namespace ab

using namespace ab;

extern "C" int ab_rotary_packed(const __nv_bfloat16* x, __nv_bfloat16* y, const int64_t* pos, const float* inv_freq,
                                int tokens, int heads, int slots, int D, int inverse, cudaStream_t st) {
  if (D % 16 != 0 || slots < 1 || heads % slots != 0 || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(y) & 15))
    return 1;
  if (tokens <= 0) return 0;
  const int grid = tokens < ab::num_sms() * 16 ? tokens : ab::num_sms() * 16;
  rotary_packed_kernel<<<grid, kRopeThreads, (D / 2) * sizeof(float2), st>>>(x, y, pos, inv_freq, tokens, heads,
                                                                           slots, D, inverse);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

static int swiglu_grid(long long n4) {
  const long long blocks = (n4 + 255) / 256;
  return (int)(blocks < ab::num_sms() * 8LL ? blocks : ab::num_sms() * 8LL);
}

extern "C" int ab_swiglu_fwd(const __nv_bfloat16* gu, __nv_bfloat16* h, long long pairs, cudaStream_t st) {
  if (pairs % 4 != 0 || (reinterpret_cast<uintptr_t>(gu) & 15) || (reinterpret_cast<uintptr_t>(h) & 7)) return 1;
  if (pairs == 0) return 0;
  swiglu_fwd_kernel<<<swiglu_grid(pairs / 4), 256, 0, st>>>(gu, h, pairs / 4);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_swiglu_bwd(const __nv_bfloat16* dh, const __nv_bfloat16* gu, __nv_bfloat16* dgu, long long pairs,
                             cudaStream_t st) {
  if (pairs % 4 != 0 || (reinterpret_cast<uintptr_t>(gu) & 15) || (reinterpret_cast<uintptr_t>(dgu) & 15) ||
      (reinterpret_cast<uintptr_t>(dh) & 7))
    return 1;
  if (pairs == 0) return 0;
  swiglu_bwd_kernel<<<swiglu_grid(pairs / 4), 256, 0, st>>>(dh, gu, dgu, pairs / 4);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
