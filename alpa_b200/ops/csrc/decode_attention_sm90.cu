// Decode-step attention with the KV-cache append fused in (K20 of SURVEY.md §2.5, OPT serving).
//
// One new token per sequence: q / k_new / v_new are [B, heads, D] views of the fused QKV projection, the caches are
// [B, S_max, heads, D], `kv_len` (device int) is the number of valid rows *including* the new one.  The kernel
//   * writes k_new / v_new into cache row kv_len-1 (replaces two strided copies + two index_copy launches),
//   * streams rows [0, kv_len) of K and V once, single pass, online softmax,
//   * merges the partial results of its 16 half-warps through shared memory, and
//   * splits the key range of one (sequence, head) over `splits` CTAs (a batch-1 decode has only `heads` independent
//     rows -- far fewer CTAs than SMs, each walking the whole context serially): every CTA
//     publishes (m, l, acc) to a workspace, the LAST CTA of the (sequence, head) to arrive merges them -- one launch.
// The op is a pure cache stream (2 * kv_len * D bf16 per head), so it runs on the CUDA cores; what matters is memory
// level parallelism: every lane keeps kUnroll K rows and kUnroll V rows (16-byte pieces) in flight.
// Because kv_len is read on the device, one captured CUDA graph serves every decode position.
// Reference behaviour: the per-token attention + cache update of examples/llm_serving/model/opt_model.py:213-300
// (dynamic_update_slice into the cache, then a masked attention over the whole cache).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "pdl.h"
#include "ptx.cuh"

namespace ab {

constexpr int kDecWarps = 8;
constexpr int kDecHalves = kDecWarps * 2;      // a half-warp (16 lanes x 16 bytes = up to 128 channels) owns one key
constexpr int kDecUnroll = 4;

__global__ void __launch_bounds__(kDecWarps * 32) decode_attention_kernel(const DecodeAttnArgs a) {
  __shared__ float sm_m[kDecHalves], sm_l[kDecHalves];
  __shared__ float sm_acc[kDecHalves][128];
  griddep_launch_dependents();
  griddep_wait();
  const int head = blockIdx.x, b = blockIdx.y, split = blockIdx.z, splits = gridDim.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int l16 = lane & 15, hw = warp * 2 + (lane >> 4);
  const int D = a.D, pieces = D >> 3;
  const bool live = l16 < pieces;                               // lanes beyond D/8 carry zeros
  const int ctx = min(*a.kv_len, a.S_max);
  const int last = ctx - 1;

  const __nv_bfloat16* kn = a.k_new + (long long)b * a.new_stride_b + (long long)head * a.new_stride_h + l16 * 8;
  const __nv_bfloat16* vn = a.v_new + (long long)b * a.new_stride_b + (long long)head * a.new_stride_h + l16 * 8;
  const long long cache_off = (long long)b * a.cache_stride_b + (long long)head * D + l16 * 8;
  const __nv_bfloat16* kc = a.k_cache + cache_off;
  const __nv_bfloat16* vc = a.v_cache + cache_off;

  float qf[8];
  {
    int4 qv = make_int4(0, 0, 0, 0);
    if (live) qv = *reinterpret_cast<const int4*>(a.q + (long long)b * a.q_stride_b + (long long)head * a.q_stride_h + l16 * 8);
    const uint32_t* qu = reinterpret_cast<const uint32_t*>(&qv);
    const float sc = a.scale * 1.4426950408889634f;             // exp2 domain
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16x2(qu[i]);
      qf[2 * i] = f.x * sc;
      qf[2 * i + 1] = f.y * sc;
    }
  }
  // this CTA's share of the keys: a multiple of 16 so that the half-warp striding below stays aligned
  const int per = ((ctx + splits - 1) / splits + kDecHalves - 1) / kDecHalves * kDecHalves;
  const int k_begin = min(split * per, ctx), k_end = min(k_begin + per, ctx);
  if (split == 0 && hw == 0 && live && last >= 0) {             // cache append
    *reinterpret_cast<int4*>(a.k_cache + cache_off + (long long)last * a.cache_stride_s) = *reinterpret_cast<const int4*>(kn);
    *reinterpret_cast<int4*>(a.v_cache + cache_off + (long long)last * a.cache_stride_s) = *reinterpret_cast<const int4*>(vn);
  }

  float m = -1e30f, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  // the trip count is uniform over the CTA (the shuffles below use the full mask)
  for (int base = k_begin; base < k_end; base += kDecHalves * kDecUnroll) {
    const int j0 = base + hw;
    int4 kv[kDecUnroll], vv[kDecUnroll];
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const int j = j0 + u * kDecHalves;
      kv[u] = make_int4(0, 0, 0, 0);
      vv[u] = make_int4(0, 0, 0, 0);
      if (live && j < k_end) {
        // the row written above is read from its source: it is not yet visible through the non-coherent path
        const __nv_bfloat16* kp = (j == last) ? kn : kc + (long long)j * a.cache_stride_s;
        const __nv_bfloat16* vp = (j == last) ? vn : vc + (long long)j * a.cache_stride_s;
        kv[u] = ld_nc_v4(kp);
        vv[u] = ld_nc_v4(vp);
      }
    }
    float s[kDecUnroll];
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const uint32_t* ku = reinterpret_cast<const uint32_t*>(&kv[u]);
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(ku[i]);
        d = fmaf(f.x, qf[2 * i], d);
        d = fmaf(f.y, qf[2 * i + 1], d);
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      s[u] = (j0 + u * kDecHalves < k_end) ? d : -INFINITY;
    }
    float mn = m;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) mn = fmaxf(mn, s[u]);
    const float alpha = ex2_approx(m - mn);
    m = mn;
    l *= alpha;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= alpha;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const float p = ex2_approx(s[u] - mn);
      l += p;
      const uint32_t* vu = reinterpret_cast<const uint32_t*>(&vv[u]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_bf16x2(vu[i]);
        acc[2 * i] = fmaf(p, f.x, acc[2 * i]);
        acc[2 * i + 1] = fmaf(p, f.y, acc[2 * i + 1]);
      }
    }
  }
  if (l16 == 0) {
    sm_m[hw] = m;
    sm_l[hw] = l;
  }
  if (live) {
#pragma unroll
    for (int i = 0; i < 8; ++i) sm_acc[hw][l16 * 8 + i] = acc[i];
  }
  __syncthreads();
  __shared__ float sm_w[kDecHalves + 1];
  __shared__ int sm_last;
  if (threadIdx.x == 0) {
    float mm = -1e30f;
#pragma unroll
    for (int h = 0; h < kDecHalves; ++h) mm = fmaxf(mm, sm_m[h]);
    float den = 0.f;
#pragma unroll
    for (int h = 0; h < kDecHalves; ++h) {
      sm_w[h] = ex2_approx(sm_m[h] - mm);
      den = fmaf(sm_l[h], sm_w[h], den);
    }
    sm_w[kDecHalves] = mm;
    sm_m[0] = den;           // reuse: CTA-level denominator
  }
  __syncthreads();
  const float cta_m = sm_w[kDecHalves], cta_den = sm_m[0];
  const long long bh = (long long)b * a.heads + head;
  if (splits == 1) {
    for (int d = threadIdx.x; d < D; d += kDecWarps * 32) {
      float num = 0.f;
#pragma unroll
      for (int h = 0; h < kDecHalves; ++h) num = fmaf(sm_acc[h][d], sm_w[h], num);
      a.o[bh * D + d] = __float2bfloat16(cta_den > 0.f ? num / cta_den : 0.f);
    }
    return;
  }
  // publish this CTA's partial: [m, den, num[D]]
  float* part = a.ws + (bh * splits + split) * (D + 2);
  for (int d = threadIdx.x; d < D; d += kDecWarps * 32) {
    float num = 0.f;
#pragma unroll
    for (int h = 0; h < kDecHalves; ++h) num = fmaf(sm_acc[h][d], sm_w[h], num);
    part[2 + d] = num;
  }
  if (threadIdx.x == 0) {
    part[0] = cta_m;
    part[1] = cta_den;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int old = atomicAdd(a.counters + bh, 1);
    sm_last = (old == splits - 1);
    if (sm_last) a.counters[bh] = 0;             // ready for the next launch (graph replay)
  }
  __syncthreads();
  if (!sm_last) return;
  __threadfence();
  const float* all = a.ws + bh * splits * (D + 2);
  float mm = -1e30f;
  for (int sp = 0; sp < splits; ++sp) mm = fmaxf(mm, __ldcg(all + sp * (D + 2)));
  for (int d = threadIdx.x; d < D; d += kDecWarps * 32) {
    float num = 0.f, den = 0.f;
    for (int sp = 0; sp < splits; ++sp) {
      const float* p = all + sp * (D + 2);
      const float w = ex2_approx(__ldcg(p) - mm);
      num = fmaf(__ldcg(p + 2 + d), w, num);
      den = fmaf(__ldcg(p + 1), w, den);
    }
    a.o[bh * D + d] = __float2bfloat16(den > 0.f ? num / den : 0.f);
  }
}

}  // namespace ab

extern "C" int ab_decode_attention(const ab::DecodeAttnArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->D % 8 != 0 || a->D < 8 || a->D > 128) return 1;
  if (a->cache_stride_s % 8 != 0 || a->cache_stride_b % 8 != 0 || a->new_stride_b % 8 != 0 || a->new_stride_h % 8 != 0 ||
      a->q_stride_b % 8 != 0 || a->q_stride_h % 8 != 0)
    return 2;                                                   // 16-byte accesses
  if (a->B <= 0 || a->heads <= 0) return 0;
  if (a->B > 65535 || a->kv_len == nullptr || a->splits < 1 || a->splits > 64) return 3;
  if (a->splits > 1 && (a->ws == nullptr || a->counters == nullptr)) return 4;
  cudaError_t e = launch_pdl(decode_attention_kernel, dim3(a->heads, a->B, a->splits), dim3(kDecWarps * 32), 0, st, *a);
  return e == cudaSuccess ? 0 : 100 + (int)e;
}
