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
// The cache is bf16, or fp8 (e4m3 rows with one fp32 scale per row and head, kv_fp8.cuh): a lane then loads 8 bytes
// per row, twice as many rows are in flight, and the scales multiply the dot product and the softmax weight instead
// of every element.
// Reference behaviour: the per-token attention + cache update of examples/llm_serving/model/opt_model.py:213-300
// (dynamic_update_slice into the cache, then a masked attention over the whole cache).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "kernels.h"
#include "kv_fp8.cuh"
#include "pdl.h"
#include "ptx.cuh"

namespace ab {

constexpr int kDecWarps = 8;
constexpr int kDecHalves = kDecWarps * 2;      // a half-warp (16 lanes x 16 bytes = up to 128 channels) owns one key
constexpr int kDecUnroll = 4;

// Rotate 8 channels [c0, c0 + 8) of one head in HF's rotate_half convention: `own` holds them, `oth` the 8 channels
// they pair with (c0 +- D/2), cs[i] = (cos, sin) of frequency i.  The expressions are rotary_packed_kernel's
// (rotary_sm90.cu), with the multiply-add contraction it compiles to written out, so both round to the same bf16.
__device__ __forceinline__ int4 rope8(int4 own, int4 oth, const float2* cs, int c0, int half) {
  const bool first = c0 < half;
  const int i0 = first ? c0 : c0 - half;
  const uint32_t* ou = reinterpret_cast<const uint32_t*>(&own);
  const uint32_t* pu = reinterpret_cast<const uint32_t*>(&oth);
  int4 r;
  uint32_t* ru = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 x = unpack_bf16x2(ou[j]), y = unpack_bf16x2(pu[j]);
    const float2 k0 = cs[i0 + 2 * j], k1 = cs[i0 + 2 * j + 1];
    // first half: x1 * c - x2 * s; second half: x2 * c + x1 * s (x is this lane's element, y its partner)
    ru[j] = first ? pack_bf16x2(__fmaf_rn(x.x, k0.x, -__fmul_rn(y.x, k0.y)), __fmaf_rn(x.y, k1.x, -__fmul_rn(y.y, k1.y)))
                  : pack_bf16x2(__fmaf_rn(x.x, k0.x, __fmul_rn(y.x, k0.y)), __fmaf_rn(x.y, k1.x, __fmul_rn(y.y, k1.y)));
  }
  return r;
}

// GC: query heads per CTA (one K/V head's group, or a chunk of it).  Every K / V row a CTA loads is used for all of
// its GC query heads.  ROPE: rotate the query heads and k_new first (the appended row is the rotated one).
// Cache: __nv_bfloat16, or __nv_fp8_e4m3 with per-row scales (the appended row is quantised here).
template <int GC, bool ROPE, typename Cache>
__global__ void __launch_bounds__(kDecWarps * 32) decode_attention_kernel(const DecodeAttnArgs a) {
  constexpr bool F8 = std::is_same_v<Cache, __nv_fp8_e4m3>;
  // K / V rows in flight per lane: registers go to the GC queries; an fp8 row piece (8 bytes) needs half the registers
  constexpr int kU = (GC <= 2 ? kDecUnroll : 2) * (F8 ? 2 : 1);
  using Piece = std::conditional_t<F8, uint2, int4>;           // one lane's 8 channels of a cache row
  __shared__ float sm_m[kDecHalves], sm_l[kDecHalves];
  __shared__ float sm_acc[kDecHalves][128];
  __shared__ float2 sm_cs[ROPE ? 64 : 1];
  griddep_launch_dependents();
  griddep_wait();
  // GC == 1 serves multi-head attention only (group == 1): blockIdx.x is the head
  const int chunks = GC == 1 ? 1 : (a.group + GC - 1) / GC;
  const int head = GC == 1 ? blockIdx.x : blockIdx.x / chunks, b = blockIdx.y, split = blockIdx.z, splits = gridDim.z;
  const int g0 = GC == 1 ? 0 : (blockIdx.x - head * chunks) * GC;        // first query head of the chunk in the group
  const int gcount = GC == 1 ? 1 : min(GC, a.group - g0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int l16 = lane & 15, hw = warp * 2 + (lane >> 4);
  const int D = a.D, pieces = D >> 3;
  const bool live = l16 < pieces;                               // lanes beyond D/8 carry zeros
  const int ctx = min(*a.kv_len, a.S_max);
  const int last = ctx - 1;
  const int half = D >> 1, poff = l16 * 8 < half ? half : -half;  // ROPE: offset of the partner channels

  if constexpr (ROPE) {
    const float p = (float)a.pos[b];
    for (int i = threadIdx.x; i < half; i += kDecWarps * 32) {
      const float ang = p * a.inv_freq[i];
      double sn, cn;
      sincos((double)ang, &sn, &cn);                            // double: see rotary_sm90.cu
      sm_cs[i] = make_float2((float)cn, (float)sn);
    }
    __syncthreads();
  }

  const __nv_bfloat16* kn = a.k_new + (long long)b * a.new_stride_b + (long long)head * a.new_stride_h + l16 * 8;
  const __nv_bfloat16* vn = a.v_new + (long long)b * a.new_stride_b + (long long)head * a.new_stride_h + l16 * 8;
  const long long cache_off = (long long)b * a.cache_stride_b + (long long)head * D + l16 * 8;
  Cache* const k_cache = static_cast<Cache*>(a.k_cache);
  Cache* const v_cache = static_cast<Cache*>(a.v_cache);
  const Cache* kc = k_cache + cache_off;
  const Cache* vc = v_cache + cache_off;
  int4 krot = make_int4(0, 0, 0, 0);                            // ROPE: the rotated new key (this lane's 8 channels)
  if constexpr (ROPE) {
    if (live) krot = rope8(*reinterpret_cast<const int4*>(kn), *reinterpret_cast<const int4*>(kn + poff), sm_cs, l16 * 8, half);
  }
  // F8: the new row quantised (amax over the half-warp's D channels); every CTA whose key range holds it attends to
  // these values, the same ones it appends
  const float* ks = nullptr;
  const float* vs = nullptr;
  Piece knew{}, vnew{};
  float ks_new = 0.f, vs_new = 0.f;
  if constexpr (F8) {
    const long long sc_off = (long long)b * a.scale_stride_b + (long long)head * a.scale_stride_h;
    ks = a.k_scale + sc_off;
    vs = a.v_scale + sc_off;
    const int4 zero = make_int4(0, 0, 0, 0);
    const int4 kraw = ROPE ? krot : live ? *reinterpret_cast<const int4*>(kn) : zero;
    const int4 vraw = live ? *reinterpret_cast<const int4*>(vn) : zero;
    float kf[8], vf[8];
    float kam = kv_bf16_unpack8(kraw, kf), vam = kv_bf16_unpack8(vraw, vf);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      kam = fmaxf(kam, __shfl_xor_sync(0xffffffffu, kam, o));
      vam = fmaxf(vam, __shfl_xor_sync(0xffffffffu, vam, o));
    }
    ks_new = kv_fp8_scale(kam);
    vs_new = kv_fp8_scale(vam);
    knew = kv_fp8_quant8(kf, ks_new);
    vnew = kv_fp8_quant8(vf, vs_new);
  }

  float qf[GC][8];
#pragma unroll
  for (int g = 0; g < GC; ++g) {
    int4 qv = make_int4(0, 0, 0, 0);
    if (live && g < gcount) {
      const __nv_bfloat16* qp = a.q + (long long)b * a.q_stride_b + (long long)head * a.q_stride_h +
                                (GC > 1 ? (long long)(g0 + g) * a.q_stride_g : 0) + l16 * 8;
      qv = *reinterpret_cast<const int4*>(qp);
      if constexpr (ROPE) qv = rope8(qv, *reinterpret_cast<const int4*>(qp + poff), sm_cs, l16 * 8, half);
    }
    const uint32_t* qu = reinterpret_cast<const uint32_t*>(&qv);
    const float sc = a.scale * 1.4426950408889634f;             // exp2 domain
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16x2(qu[i]);
      qf[g][2 * i] = f.x * sc;
      qf[g][2 * i + 1] = f.y * sc;
    }
  }
  // this CTA's share of the keys: a multiple of 16 so that the half-warp striding below stays aligned
  const int per = ((ctx + splits - 1) / splits + kDecHalves - 1) / kDecHalves * kDecHalves;
  const int k_begin = min(split * per, ctx), k_end = min(k_begin + per, ctx);
  if (split == 0 && hw == 0 && live && last >= 0 && g0 == 0) {  // cache append (once per K/V head)
    if constexpr (F8) {
      *reinterpret_cast<uint2*>(k_cache + cache_off + (long long)last * a.cache_stride_s) = knew;
      *reinterpret_cast<uint2*>(v_cache + cache_off + (long long)last * a.cache_stride_s) = vnew;
      if (l16 == 0) {
        a.k_scale[(long long)b * a.scale_stride_b + (long long)head * a.scale_stride_h + last] = ks_new;
        a.v_scale[(long long)b * a.scale_stride_b + (long long)head * a.scale_stride_h + last] = vs_new;
      }
    } else {
      *reinterpret_cast<int4*>(k_cache + cache_off + (long long)last * a.cache_stride_s) =
          ROPE ? krot : *reinterpret_cast<const int4*>(kn);
      *reinterpret_cast<int4*>(v_cache + cache_off + (long long)last * a.cache_stride_s) = *reinterpret_cast<const int4*>(vn);
    }
  }

  float m[GC], l[GC], acc[GC][8];
#pragma unroll
  for (int g = 0; g < GC; ++g) {
    m[g] = -1e30f;
    l[g] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[g][i] = 0.f;
  }

  // the trip count is uniform over the CTA (the shuffles below use the full mask)
  for (int base = k_begin; base < k_end; base += kDecHalves * kU) {
    const int j0 = base + hw;
    Piece kv[kU], vv[kU];
    float ksc[F8 ? kU : 1], vsc[F8 ? kU : 1];                    // F8: the rows' scales
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int j = j0 + u * kDecHalves;
      if constexpr (F8) {
        kv[u] = make_uint2(0, 0);
        vv[u] = make_uint2(0, 0);
        ksc[u] = vsc[u] = 0.f;
        if (live && j < k_end) {
          if (j == last) {
            kv[u] = knew;
            vv[u] = vnew;
            ksc[u] = ks_new;
            vsc[u] = vs_new;
          } else {
            kv[u] = ld_nc_v2(kc + (long long)j * a.cache_stride_s);
            vv[u] = ld_nc_v2(vc + (long long)j * a.cache_stride_s);
            ksc[u] = __ldg(ks + j);
            vsc[u] = __ldg(vs + j);
          }
        }
      } else {
        kv[u] = make_int4(0, 0, 0, 0);
        vv[u] = make_int4(0, 0, 0, 0);
        if (live && j < k_end) {
          // the row written above is read from its source: it is not yet visible through the non-coherent path
          if constexpr (ROPE) {
            kv[u] = (j == last) ? krot : ld_nc_v4(kc + (long long)j * a.cache_stride_s);
          } else {
            const __nv_bfloat16* kp = (j == last) ? kn : kc + (long long)j * a.cache_stride_s;
            kv[u] = ld_nc_v4(kp);
          }
          const __nv_bfloat16* vp = (j == last) ? vn : vc + (long long)j * a.cache_stride_s;
          vv[u] = ld_nc_v4(vp);
        }
      }
    }
    float s[GC][kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      if constexpr (F8) {
        float kf[8];
        kv_fp8_unpack8(kv[u], kf);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          float d = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) d = fmaf(kf[i], qf[g][i], d);
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
          s[g][u] = (j0 + u * kDecHalves < k_end) ? d * ksc[u] : -INFINITY;   // score = s_k * dot(q, k8)
        }
      } else {
        const uint32_t* ku = reinterpret_cast<const uint32_t*>(&kv[u]);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          float d = 0.f;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = unpack_bf16x2(ku[i]);
            d = fmaf(f.x, qf[g][2 * i], d);
            d = fmaf(f.y, qf[g][2 * i + 1], d);
          }
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
          s[g][u] = (j0 + u * kDecHalves < k_end) ? d : -INFINITY;
        }
      }
    }
#pragma unroll
    for (int g = 0; g < GC; ++g) {
      float mn = m[g];
#pragma unroll
      for (int u = 0; u < kU; ++u) mn = fmaxf(mn, s[g][u]);
      const float alpha = ex2_approx(m[g] - mn);
      m[g] = mn;
      l[g] *= alpha;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[g][i] *= alpha;
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      if constexpr (F8) {
        float vf[8];
        kv_fp8_unpack8(vv[u], vf);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          const float p = ex2_approx(s[g][u] - m[g]);
          l[g] += p;
          const float pv = p * vsc[u];                          // acc += (p * s_v) * v8
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[g][i] = fmaf(pv, vf[i], acc[g][i]);
        }
      } else {
        const uint32_t* vu = reinterpret_cast<const uint32_t*>(&vv[u]);
#pragma unroll
        for (int g = 0; g < GC; ++g) {
          const float p = ex2_approx(s[g][u] - m[g]);
          l[g] += p;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = unpack_bf16x2(vu[i]);
            acc[g][2 * i] = fmaf(p, f.x, acc[g][2 * i]);
            acc[g][2 * i + 1] = fmaf(p, f.y, acc[g][2 * i + 1]);
          }
        }
      }
    }
  }
  __shared__ float sm_w[kDecHalves + 1];
  __shared__ int sm_last;
  // rows of the workspace / counters: one per CTA row (sequence, K/V head, chunk)
  const long long row = GC == 1 ? (long long)b * a.heads + head : (long long)b * gridDim.x + blockIdx.x;
  const int q0 = GC == 1 ? head : head * a.group + g0;          // first query head of this CTA
  // merge the 16 half-warps, one query head after the other through the same shared buffers
#pragma unroll
  for (int g = 0; g < GC; ++g) {
    if (GC > 1) __syncthreads();                                // the previous head's readers are done
    if (l16 == 0) {
      sm_m[hw] = m[g];
      sm_l[hw] = l[g];
    }
    if (live) {
#pragma unroll
      for (int i = 0; i < 8; ++i) sm_acc[hw][l16 * 8 + i] = acc[g][i];
    }
    __syncthreads();
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
    if (splits == 1) {
      if (g < gcount) {
        const long long bh = (long long)b * a.heads + q0 + g;
        for (int d = threadIdx.x; d < D; d += kDecWarps * 32) {
          float num = 0.f;
#pragma unroll
          for (int h = 0; h < kDecHalves; ++h) num = fmaf(sm_acc[h][d], sm_w[h], num);
          a.o[bh * D + d] = __float2bfloat16(cta_den > 0.f ? num / cta_den : 0.f);
        }
      }
      if (GC == 1) return;
      continue;
    }
    // publish this CTA's partial of head g: [m, den, num[D]]
    float* part = a.ws + ((row * splits + split) * GC + g) * (D + 2);
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
  }
  if (GC > 1 && splits == 1) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int old = atomicAdd(a.counters + row, 1);
    sm_last = (old == splits - 1);
    if (sm_last) a.counters[row] = 0;            // ready for the next launch (graph replay)
  }
  __syncthreads();
  if (!sm_last) return;
  __threadfence();
#pragma unroll 1
  for (int g = 0; g < gcount; ++g) {
    const float* all = a.ws + row * splits * GC * (D + 2) + g * (D + 2);
    float mm = -1e30f;
    for (int sp = 0; sp < splits; ++sp) mm = fmaxf(mm, __ldcg(all + sp * GC * (D + 2)));
    const long long bh = (long long)b * a.heads + q0 + g;
    for (int d = threadIdx.x; d < D; d += kDecWarps * 32) {
      float num = 0.f, den = 0.f;
      for (int sp = 0; sp < splits; ++sp) {
        const float* p = all + sp * GC * (D + 2);
        const float w = ex2_approx(__ldcg(p) - mm);
        num = fmaf(__ldcg(p + 2 + d), w, num);
        den = fmaf(__ldcg(p + 1), w, den);
      }
      a.o[bh * D + d] = __float2bfloat16(den > 0.f ? num / den : 0.f);
    }
  }
}

// query heads per CTA: the whole group up to 8 (register budget), else chunks of 8 that each re-read the rows
static int decode_chunk(int group) { return group == 1 ? 1 : group == 2 ? 2 : group <= 4 ? 4 : 8; }

template <int GC, typename Cache>
static cudaError_t decode_launch(const DecodeAttnArgs& a, dim3 grid, cudaStream_t st) {
  if (a.pos != nullptr) return launch_pdl(decode_attention_kernel<GC, true, Cache>, grid, dim3(kDecWarps * 32), 0, st, a);
  return launch_pdl(decode_attention_kernel<GC, false, Cache>, grid, dim3(kDecWarps * 32), 0, st, a);
}

template <int GC>
static cudaError_t decode_launch(const DecodeAttnArgs& a, dim3 grid, cudaStream_t st) {
  return a.cache_fp8 ? decode_launch<GC, __nv_fp8_e4m3>(a, grid, st) : decode_launch<GC, __nv_bfloat16>(a, grid, st);
}

}  // namespace ab

extern "C" int ab_decode_attention_chunk(const ab::DecodeAttnArgs* a) { return ab::decode_chunk(a->group); }
extern "C" int ab_decode_attention_rows(const ab::DecodeAttnArgs* a) {
  const int gc = ab::decode_chunk(a->group);
  return a->kv_heads * ((a->group + gc - 1) / gc);
}

extern "C" int ab_decode_attention(const ab::DecodeAttnArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->D % 8 != 0 || a->D < 8 || a->D > 128) return 1;
  if (a->cache_stride_s % 8 != 0 || a->cache_stride_b % 8 != 0 || a->new_stride_b % 8 != 0 || a->new_stride_h % 8 != 0 ||
      a->q_stride_b % 8 != 0 || a->q_stride_h % 8 != 0 || a->q_stride_g % 8 != 0)
    return 2;                                                   // 16-byte accesses
  if (a->B <= 0 || a->heads <= 0) return 0;
  if (a->B > 65535 || a->kv_len == nullptr || a->splits < 1 || a->splits > 64) return 3;
  if (a->splits > 1 && (a->ws == nullptr || a->counters == nullptr)) return 4;
  if (a->group < 1 || a->kv_heads < 1 || a->heads != a->kv_heads * a->group) return 5;
  if ((a->pos == nullptr) != (a->inv_freq == nullptr) || (a->pos != nullptr && a->D % 16 != 0)) return 6;
  if (a->cache_fp8 && (a->k_scale == nullptr || a->v_scale == nullptr)) return 7;
  const dim3 grid(ab_decode_attention_rows(a), a->B, a->splits);
  cudaError_t e;
  switch (decode_chunk(a->group)) {
    case 1: e = decode_launch<1>(*a, grid, st); break;
    case 2: e = decode_launch<2>(*a, grid, st); break;
    case 4: e = decode_launch<4>(*a, grid, st); break;
    default: e = decode_launch<8>(*a, grid, st); break;
  }
  return e == cudaSuccess ? 0 : 100 + (int)e;
}
