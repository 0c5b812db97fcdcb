// Masked multi-head attention over a ragged 1-D token batch (iteration-level batching for serving).
//
// Reference behaviour: examples/llm_serving/model/opt_model_1d.py:151-178 calls the external FasterTransformer
// `fused_mmha(qkv, bias, cache_k, cache_v)` on a flat token batch whose tokens belong to different sequences.
//
// Layout here: q/o are [T, heads, D]; the KV cache is [slots, heads / group, D] (grouped-query attention: query head h
// reads cache head h / group; group = 1 is multi-head attention).  Token t attends to keys j < ctx_len[t] of its
// sequence -- prompt tokens and decode tokens look the same, causality is encoded in ctx_len.  Key j lives in cache row
//   contiguous  seq_start[t] + j                 (every sequence owns a slot range, KVCacheManager)
//   paged       (bt[j >> log2 bs] << log2 bs) | (j & (bs - 1)), bt = row seq_start[t] of the block table
//               (fixed-size blocks handed out on demand, PagedKVCacheManager; alpa_b200/csrc/serving_runtime.cpp)
// The paged instantiation only changes where a key's row is: scores, softmax, the order of the P*V sums and the ALiBi
// bias (by logical position j) are the contiguous kernel's, so both give the same bits on the same keys.
// One CTA per (head, token):
//   pass 1  thread-per-key dot products with 16-byte K loads -> scores in shared memory, block max / sum
//   pass 2  thread-per-channel-pair accumulation of P*V with coalesced 4-byte V loads, key range split over groups
// The op is bandwidth bound (it streams the sequence's K and V once per query token), so it stays on the CUDA cores.
// The cache is bf16, or fp8 (e4m3 rows with one fp32 scale per row and cache head, kv_fp8.cuh): 8-byte K loads in
// pass 1, 2-byte V loads in pass 2, and the scales multiply the dot product and the softmax weight.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "kernels.h"
#include "kv_fp8.cuh"

namespace ab {

constexpr int kRaggedThreads = 128;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename Cache, bool Paged>
__global__ void __launch_bounds__(kRaggedThreads) ragged_attention_kernel(RaggedAttnArgs a) {
  constexpr bool F8 = std::is_same_v<Cache, __nv_fp8_e4m3>;
  extern __shared__ __align__(16) float smem[];
  const int head = blockIdx.x, t = blockIdx.y, tid = threadIdx.x;
  const int D = a.D;
  float* qs = smem;                 // [D]
  float* red = qs + D;              // [8]
  float* part = red + 8;            // [groups][D]
  const int half = D / 2;
  const int groups = kRaggedThreads / half;
  float* sc = part + groups * D;    // [ctx]

  const int ctx = min(a.ctx_len[t], a.max_ctx);
  __nv_bfloat16* o = a.o + (long long)t * a.o_stride_t + (long long)head * D;
  if (ctx <= 0) {                   // padding token
    for (int d = tid; d < D; d += kRaggedThreads) o[d] = __float2bfloat16(0.f);
    return;
  }
  // contiguous: rows are row0 + j.  paged: row0 = 0 and key j's row comes from the sequence's block table row
  const long long row0 = Paged ? 0 : a.seq_start[t];
  const int* bt = Paged ? a.block_table + (long long)a.seq_start[t] * a.bt_stride : nullptr;
  const int lg = a.block_log2;
  const __nv_bfloat16* q = a.q + (long long)t * a.q_stride_t + (long long)head * a.q_stride_h;
  for (int d = tid; d < D; d += kRaggedThreads) qs[d] = __bfloat162float(q[d]) * a.scale;
  __syncthreads();

  const float slope = a.alibi ? a.alibi[head] : 0.f;
  const int kv_head = head / a.group;
  const Cache* kbase = static_cast<const Cache*>(a.k_cache) + row0 * a.kv_stride_s + (long long)kv_head * D;
  const float* ks = F8 ? a.k_scale + kv_head * a.scale_stride_h + row0 : nullptr;
  const float* vs = F8 ? a.v_scale + kv_head * a.scale_stride_h + row0 : nullptr;
  float lmax = -INFINITY;
  for (int j = tid; j < ctx; j += kRaggedThreads) {
    float s = 0.f;
    long long r = j;
    if constexpr (Paged) r = ((long long)__ldg(bt + (j >> lg)) << lg) | (j & ((1 << lg) - 1));
    if constexpr (F8) {
      const uint2* kr = reinterpret_cast<const uint2*>(kbase + r * a.kv_stride_s);
      for (int c = 0; c < D / 8; ++c) {
        float f[8];
        kv_fp8_unpack8(__ldg(kr + c), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) s = fmaf(f[e], qs[c * 8 + e], s);
      }
      s *= __ldg(ks + r);                                       // score = s_k * dot(q, k8)
    } else {
      const int4* kr = reinterpret_cast<const int4*>(kbase + r * a.kv_stride_s);
      for (int c = 0; c < D / 8; ++c) {
        int4 pk = __ldg(kr + c);
        const __nv_bfloat162* k2 = reinterpret_cast<const __nv_bfloat162*>(&pk);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __bfloat1622float2(k2[e]);
          s = fmaf(f.x, qs[c * 8 + 2 * e], s);
          s = fmaf(f.y, qs[c * 8 + 2 * e + 1], s);
        }
      }
    }
    s += slope * (float)j;
    sc[j] = s;
    lmax = fmaxf(lmax, s);
  }
  lmax = warp_max(lmax);
  if ((tid & 31) == 0) red[tid >> 5] = lmax;
  __syncthreads();
  const float m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  float lsum = 0.f;
  for (int j = tid; j < ctx; j += kRaggedThreads) {
    float e = __expf(sc[j] - m);
    sc[j] = e;
    lsum += e;
  }
  lsum = warp_sum(lsum);
  if ((tid & 31) == 0) red[4 + (tid >> 5)] = lsum;
  __syncthreads();                   // also publishes sc[]
  const float inv = 1.f / (red[4] + red[5] + red[6] + red[7]);

  const int g = tid / half, c = tid - g * half;
  if (g < groups) {
    const Cache* vbase = static_cast<const Cache*>(a.v_cache) + row0 * a.kv_stride_s + (long long)kv_head * D + 2 * c;
    float acc0 = 0.f, acc1 = 0.f;
    // paged: a thread steps through keys in order, so it keeps its current block's first row in a register and
    // reads the table only when it enters the next block
    int cur_blk = -1;
    long long blk_row = 0;
    for (int j = g; j < ctx; j += groups) {
      float2 f;
      float p = sc[j];
      long long r = j;
      if constexpr (Paged) {
        if ((j >> lg) != cur_blk) {
          cur_blk = j >> lg;
          blk_row = (long long)__ldg(bt + cur_blk) << lg;
        }
        r = blk_row | (j & ((1 << lg) - 1));
      }
      if constexpr (F8) {
        f = kv_fp8_unpack2(*reinterpret_cast<const uint16_t*>(vbase + r * a.kv_stride_s));
        p *= __ldg(vs + r);                                     // acc += (p * s_v) * v8
      } else {
        f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(vbase + r * a.kv_stride_s));
      }
      acc0 = fmaf(p, f.x, acc0);
      acc1 = fmaf(p, f.y, acc1);
    }
    part[g * D + 2 * c] = acc0;
    part[g * D + 2 * c + 1] = acc1;
  }
  __syncthreads();
  for (int d = tid; d < D; d += kRaggedThreads) {
    float s = 0.f;
    for (int gg = 0; gg < groups; ++gg) s += part[gg * D + d];
    o[d] = __float2bfloat16(s * inv);
  }
}

}  // namespace ab

extern "C" int ab_ragged_attention(const ab::RaggedAttnArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->D % 8 != 0 || a->D < 16 || a->D > 256) return 1;       // 16-byte K loads, channel pairs in pass 2
  if (a->kv_stride_s % 8 != 0 || a->q_stride_t % 2 != 0) return 2;
  if (a->T <= 0) return 0;
  if (a->T > 65535 || a->max_ctx <= 0) return 5;
  if (a->group < 1 || a->heads % a->group != 0) return 6;
  const int half = a->D / 2, groups = kRaggedThreads / half;
  if (groups < 1) return 3;
  const size_t smem = sizeof(float) * ((size_t)a->D + 8 + (size_t)groups * a->D + (size_t)a->max_ctx);
  if (smem > 200 * 1024) return 4;
  if (a->cache_fp8 && (a->k_scale == nullptr || a->v_scale == nullptr)) return 7;
  const bool paged = a->block_table != nullptr;
  if (paged && (a->block_log2 < 0 || a->block_log2 > 10 || a->bt_stride < ((long long)a->max_ctx + (1 << a->block_log2) - 1) >> a->block_log2))
    return 8;
  auto kernel = a->cache_fp8 ? (paged ? ragged_attention_kernel<__nv_fp8_e4m3, true> : ragged_attention_kernel<__nv_fp8_e4m3, false>)
                             : (paged ? ragged_attention_kernel<__nv_bfloat16, true> : ragged_attention_kernel<__nv_bfloat16, false>);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return 100 + (int)e;
  }
  dim3 grid(a->heads, a->T);
  kernel<<<grid, kRaggedThreads, smem, st>>>(*a);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : 100 + (int)e;
}
