// Store into and load from the fp8 KV cache (format: kv_fp8.cuh).
//
// Store: bf16 K / V rows, read straight from strided views of the packed QKV projection, are quantised into cache
// rows (a prompt's rows b * S + start + t, or the slots of a ragged batch).  One warp per (token, head) of K or V: each
// lane holds 8 channels, the row's amax is a warp reduction, and the lane writes its 8 bytes; lane 0 the scale.
// Load: rows [0, end) of every sequence dequantised into a bf16 scratch, bf16(float(q) * s), for the prefill's
// attention kernel (which reads bf16 K / V).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "kv_fp8.cuh"
#include "ptx.cuh"

namespace ab {

constexpr int kKVThreads = 256;

__global__ void __launch_bounds__(kKVThreads) kv_cache_store_kernel(const KVStoreArgs a) {
  const long long item = ((long long)blockIdx.x * kKVThreads + threadIdx.x) >> 5;  // (token, head, K or V)
  const int lane = threadIdx.x & 31;
  const long long tokens = (long long)a.B * a.T;
  if (item >= tokens * a.H * 2) return;                        // uniform over the warp
  const bool is_v = item >= tokens * a.H;
  const long long th = is_v ? item - tokens * a.H : item;
  const int h = (int)(th % a.H);
  const long long n = th / a.H;
  const int b = (int)(n / a.T), t = (int)(n % a.T);
  const bool live = lane * 8 < a.D;
  const long long* st = is_v ? a.v_stride : a.k_stride;
  const __nv_bfloat16* src = (is_v ? a.v : a.k) + b * st[0] + t * st[1] + h * st[2] + lane * 8;
  float x[8];
  float amax = kv_bf16_unpack8(live ? *reinterpret_cast<const int4*>(src) : make_int4(0, 0, 0, 0), x);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float s = kv_fp8_scale(amax);
  const long long r = a.rows != nullptr ? a.rows[n] : (long long)b * a.S + a.start + t;
  if (r < 0 || r >= a.cache_rows) return;                     // uniform over the warp
  if (live) {
    uint8_t* dst = (is_v ? a.v_data : a.k_data) + (r * a.H + h) * a.D + lane * 8;
    *reinterpret_cast<uint2*>(dst) = kv_fp8_quant8(x, s);
  }
  if (lane == 0) (is_v ? a.v_scale : a.k_scale)[(r / a.S) * a.scale_stride_b + h * a.scale_stride_h + r % a.S] = s;
}

__global__ void __launch_bounds__(kKVThreads) kv_cache_load_kernel(const uint8_t* data, const float* scale,
                                                                   __nv_bfloat16* out, int end, int H, int D,
                                                                   long long data_stride_b, long long scale_stride_b,
                                                                   long long scale_stride_h, long long pieces) {
  const long long i = (long long)blockIdx.x * kKVThreads + threadIdx.x;   // one 8-channel piece of out
  if (i >= pieces) return;
  const int per_row = D / 8;
  const int c = (int)(i % per_row);
  const long long bsh = i / per_row;                           // (b, s, h) of out [B, end, H, D]
  const int h = (int)(bsh % H);
  const long long bs = bsh / H;
  const int s = (int)(bs % end), b = (int)(bs / end);
  const float sc = scale[b * scale_stride_b + h * scale_stride_h + s];
  float f[8];
  kv_fp8_unpack8(*reinterpret_cast<const uint2*>(data + b * data_stride_b + ((long long)s * H + h) * D + c * 8), f);
  int4 o;
  uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
  for (int k = 0; k < 4; ++k) ou[k] = pack_bf16x2(__fmul_rn(f[2 * k], sc), __fmul_rn(f[2 * k + 1], sc));
  *reinterpret_cast<int4*>(out + i * 8) = o;
}

}  // namespace ab

extern "C" int ab_kv_cache_store(const ab::KVStoreArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->D % 8 != 0 || a->D < 8 || a->D > 256) return 1;
  for (int i = 0; i < 3; ++i)
    if (a->k_stride[i] % 8 != 0 || a->v_stride[i] % 8 != 0) return 2;  // 16-byte loads
  if (a->S <= 0 || a->H <= 0) return 3;
  const long long warps = (long long)a->B * a->T * a->H * 2;
  if (warps == 0) return 0;
  const long long blocks = (warps * 32 + kKVThreads - 1) / kKVThreads;
  if (blocks > 0x7fffffffLL) return 4;
  kv_cache_store_kernel<<<(unsigned)blocks, kKVThreads, 0, st>>>(*a);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : 100 + (int)e;
}

extern "C" int ab_kv_cache_load(const uint8_t* data, const float* scale, __nv_bfloat16* out, int B, int end, int H,
                                int D, long long data_stride_b, long long scale_stride_b, long long scale_stride_h,
                                cudaStream_t st) {
  using namespace ab;
  if (D % 8 != 0 || D < 8) return 1;
  if (data_stride_b % 8 != 0) return 2;
  const long long pieces = (long long)B * end * H * (D / 8);
  if (pieces == 0) return 0;
  const long long blocks = (pieces + kKVThreads - 1) / kKVThreads;
  if (blocks > 0x7fffffffLL) return 4;
  kv_cache_load_kernel<<<(unsigned)blocks, kKVThreads, 0, st>>>(data, scale, out, end, H, D, data_stride_b,
                                                                 scale_stride_b, scale_stride_h, pieces);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : 100 + (int)e;
}
