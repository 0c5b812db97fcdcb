// Counter-based (Philox4x32-10) dropout: the keep decision of an element depends only on (seed, stream, GLOBAL linear
// index), never on how the tensor is sharded or which device runs it.  A sharded execution therefore produces exactly
// the mask of the single-device run, the backward pass regenerates the mask instead of storing it, and a rematerialised
// forward reproduces its first execution.
//
// Reference behaviour: alpa replaces jax's threefry by XLA's stateful RngUniform with a per-device seed
// (alpa/monkey_patch.py:52-160, K19/K22 of SURVEY §2.5); masks there differ between parallel plans.
//
// Random word of global index g: lane (g & 3) of Philox(counter = {lo(g>>2), hi(g>>2), stream, 0}, key = seed).
// Fast path: 4 consecutive elements of the last dim share one Philox call (needs 4 | local last dim, offset and
// global last dim); otherwise one call per element.  bf16 and fp32 payloads.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace ab {

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                              uint32_t k1, uint32_t out[4]) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

template <typename T>
__device__ __forceinline__ float ld(const T* p);
template <>
__device__ __forceinline__ float ld<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T>
__device__ __forceinline__ void st(T* p, float v);
template <>
__device__ __forceinline__ void st<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void st<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

// global linear index of the local linear index `i`
__device__ __forceinline__ unsigned long long global_index(const DropoutArgs& a, long long i) {
  unsigned long long g = 0;
#pragma unroll
  for (int d = kDropoutMaxDims - 1; d >= 0; --d) {
    if (d >= a.ndim) continue;
    const long long c = i % a.local_shape[d];
    i /= a.local_shape[d];
    g += (unsigned long long)(c + a.offset[d]) * (unsigned long long)a.global_stride[d];
  }
  return g;
}

template <typename T, bool VEC4>
__global__ void __launch_bounds__(256) dropout_kernel(DropoutArgs a) {
  const unsigned long long seed = *a.seed;
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const T* x = reinterpret_cast<const T*>(a.x);
  T* y = reinterpret_cast<T*>(a.y);
  const long long stride = (long long)gridDim.x * blockDim.x;
  if (VEC4) {
    const long long groups = a.numel / 4;
    for (long long gi = (long long)blockIdx.x * blockDim.x + threadIdx.x; gi < groups; gi += stride) {
      const long long i = gi * 4;
      const unsigned long long g = global_index(a, i);          // multiple of 4 by construction
      uint32_t r[4];
      philox4x32_10((uint32_t)(g >> 2), (uint32_t)(g >> 34), a.stream, 0u, k0, k1, r);
#pragma unroll
      for (int e = 0; e < 4; ++e) st<T>(y + i + e, r[e] >= a.threshold ? ld<T>(x + i + e) * a.scale : 0.f);
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.numel; i += stride) {
      const unsigned long long g = global_index(a, i);
      uint32_t r[4];
      philox4x32_10((uint32_t)(g >> 2), (uint32_t)(g >> 34), a.stream, 0u, k0, k1, r);
      st<T>(y + i, r[g & 3] >= a.threshold ? ld<T>(x + i) * a.scale : 0.f);
    }
  }
}

}  // namespace ab

extern "C" int ab_dropout(const ab::DropoutArgs* a, int is_bf16, cudaStream_t st) {
  using namespace ab;
  if (a->ndim < 1 || a->ndim > kDropoutMaxDims) return 1;
  if (a->numel <= 0) return 0;
  const int last = a->ndim - 1;
  const bool vec4 = a->local_shape[last] % 4 == 0 && a->offset[last] % 4 == 0 && a->global_stride[last] == 1 &&
                    (a->ndim == 1 || a->global_stride[last - 1] % 4 == 0);
  const long long work = vec4 ? a->numel / 4 : a->numel;
  const int block = 256;
  long long blocks = (work + block - 1) / block;
  if (blocks > (long long)ab::num_sms() * 16) blocks = (long long)ab::num_sms() * 16;
  if (is_bf16) {
    if (vec4) dropout_kernel<__nv_bfloat16, true><<<(int)blocks, block, 0, st>>>(*a);
    else dropout_kernel<__nv_bfloat16, false><<<(int)blocks, block, 0, st>>>(*a);
  } else {
    if (vec4) dropout_kernel<float, true><<<(int)blocks, block, 0, st>>>(*a);
    else dropout_kernel<float, false><<<(int)blocks, block, 0, st>>>(*a);
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : 100 + (int)e;
}
