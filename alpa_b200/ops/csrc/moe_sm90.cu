// Mixture-of-experts routing kernels for sm_90a: GShard top-2 routing, token dispatch and combine.
//
// The dispatch/combine kernels address the expert buffers through a small table of base pointers, one per
// expert-parallel peer: with a single entry they are the local scatter/gather; with one entry per GPU of an
// NVLink domain (symmetric-memory mappings of every peer's buffer) the same kernels *are* the all-to-all --
// tokens are stored straight into the owning GPU's expert buffer / read straight from it, so no separate
// collective (and no send/recv staging copy) runs.  Reference semantics: alpa/model/moe.py:85-186 (dense
// one-hot einsum formulation) and the all-to-all the XLA SPMD partitioner inserts around it.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "ptx.cuh"

namespace ab {

namespace {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr int kRouteThreads = 1024;
constexpr int kRouteWarps = kRouteThreads / 32;
constexpr int kMaxExperts = 256;

// One CTA per group.  Position of a token inside its expert = number of earlier tokens (in sequence order)
// routed to the same expert: warp-level match + per-warp histogram + scan over warps, chunk by chunk.
__global__ void __launch_bounds__(kRouteThreads)
moe_top2_route_kernel(const float* __restrict__ gates, int64_t* __restrict__ expert, int64_t* __restrict__ slot,
                      int S, int E, int C) {
  __shared__ int hist[kRouteWarps][kMaxExperts];   // per-warp counts of the current chunk (then prefixes)
  __shared__ int base[kMaxExperts];                // running count per expert
  const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* gg = gates + (size_t)g * S * E;
  int64_t* ex = expert + (size_t)g * S * 2;
  int64_t* sl = slot + (size_t)g * S * 2;
  // ---- top-2 experts of every token
  for (int s = tid; s < S; s += kRouteThreads) {
    const float* row = gg + (size_t)s * E;
    float b1 = -INFINITY;
    int i1 = 0;
    for (int e = 0; e < E; ++e) {
      const float v = row[e];
      if (v > b1) {
        b1 = v; i1 = e;
      }
    }
    // second choice: argmax of the gates with the first choice's gate replaced by 0 (first index of the maximum).
    // fp32 softmax underflows to exact zeros, so this can pick i1 again, as the dense top2_gating does.
    float b2 = -INFINITY;
    int i2 = 0;
    for (int e = 0; e < E; ++e) {
      const float v = e == i1 ? 0.f : row[e];
      if (v > b2) {
        b2 = v; i2 = e;
      }
    }
    ex[2 * s] = i1;
    ex[2 * s + 1] = i2;
  }
  for (int e = tid; e < E; e += kRouteThreads) base[e] = 0;
  __syncthreads();
  for (int choice = 0; choice < 2; ++choice) {
    for (int s0 = 0; s0 < S; s0 += kRouteThreads) {
      for (int i = tid; i < kRouteWarps * E; i += kRouteThreads) hist[i / E][i % E] = 0;
      __syncthreads();
      const int s = s0 + tid;
      const bool valid = s < S;
      const int e = valid ? (int)ex[2 * s + choice] : -1;
      const unsigned mask = __match_any_sync(0xffffffffu, e);
      const int rank = __popc(mask & ((1u << lane) - 1u));
      if (valid && rank == 0) hist[warp][e] = __popc(mask);
      __syncthreads();
      // exclusive scan over warps, one thread per expert
      for (int ee = tid; ee < E; ee += kRouteThreads) {
        int run = base[ee];
        for (int w = 0; w < kRouteWarps; ++w) {
          const int c = hist[w][ee];
          hist[w][ee] = run;
          run += c;
        }
        base[ee] = run;
      }
      __syncthreads();
      if (valid) {
        const int pos = hist[warp][e] + rank;
        sl[2 * s + choice] = pos < C ? pos : -1;
      }
      __syncthreads();
    }
    // second choices continue after the *kept* first choices
    for (int e = tid; e < E; e += kRouteThreads) base[e] = min(base[e], C);
    __syncthreads();
  }
}

// warp per (token, choice): d[peer(e)][e_local, (g_off + g) * C + c, :] = w * x[g, s, :]
__global__ void __launch_bounds__(256)
moe_dispatch_kernel(const __nv_bfloat16* __restrict__ x, const int64_t* __restrict__ expert,
                    const int64_t* __restrict__ slot, const __nv_bfloat16* __restrict__ weight, MoePeers dst,
                    int GS, int S, int K, int M, int C, int g_off, int G_total) {
  const int lane = threadIdx.x & 31;
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wid >= (long long)GS * K) return;
  const long long tok = wid / K;
  const int64_t c = slot[wid];
  if (c < 0) return;
  const int e = (int)expert[wid];
  const int g = (int)(tok / S);
  const int peer = e / dst.experts_per_peer, el = e % dst.experts_per_peer;
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(dst.ptr[peer]) +
                       ((size_t)el * G_total * C + (size_t)(g_off + g) * C + c) * M;
  const __nv_bfloat16* in = x + (size_t)tok * M;
  const float w = weight ? __bfloat162float(weight[wid]) : 1.f;
  for (int i = lane * 8; i < M; i += 256) {
    int4 v = ld_nc_v4(in + i);
    if (weight) {
      uint32_t* u = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        u[j] = pack_bf16x2(f.x * w, f.y * w);
      }
    }
    *reinterpret_cast<int4*>(out + i) = v;
  }
}

// warp per token: out[g, s, :] = sum_k w_k * eo[peer(e_k)][e_local, (g_off + g) * C + c_k, :]
__global__ void __launch_bounds__(256)
moe_combine_kernel(MoePeers src, const int64_t* __restrict__ expert, const int64_t* __restrict__ slot,
                   const __nv_bfloat16* __restrict__ weight, __nv_bfloat16* __restrict__ out, int GS, int S, int K,
                   int M, int C, int g_off, int G_total) {
  const int lane = threadIdx.x & 31;
  const long long tok = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (tok >= GS) return;
  const int g = (int)(tok / S);
  for (int i = lane * 8; i < M; i += 256) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < K; ++k) {
      const int64_t c = slot[tok * K + k];
      if (c < 0) continue;
      const int e = (int)expert[tok * K + k];
      const int peer = e / src.experts_per_peer, el = e % src.experts_per_peer;
      const __nv_bfloat16* row = reinterpret_cast<const __nv_bfloat16*>(src.ptr[peer]) +
                                 ((size_t)el * G_total * C + (size_t)(g_off + g) * C + c) * M;
      const float w = weight ? __bfloat162float(weight[tok * K + k]) : 1.f;
      const int4 v = *reinterpret_cast<const int4*>(row + i);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        acc[2 * j] += w * f.x;
        acc[2 * j + 1] += w * f.y;
      }
    }
    int4 o;
    uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) ou[j] = pack_bf16x2(acc[2 * j], acc[2 * j + 1]);
    *reinterpret_cast<int4*>(out + (size_t)tok * M + i) = o;
  }
}

// warp per (token, choice): dw[g, s, k] = <dout[g, s, :], eo[e, g*C + c, :]>
__global__ void __launch_bounds__(256)
moe_combine_wgrad_kernel(const __nv_bfloat16* __restrict__ dout, MoePeers src, const int64_t* __restrict__ expert,
                         const int64_t* __restrict__ slot, __nv_bfloat16* __restrict__ dw, int GS, int S, int K,
                         int M, int C, int g_off, int G_total) {
  const int lane = threadIdx.x & 31;
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wid >= (long long)GS * K) return;
  const long long tok = wid / K;
  const int64_t c = slot[wid];
  float acc = 0.f;
  if (c >= 0) {
    const int e = (int)expert[wid];
    const int g = (int)(tok / S);
    const int peer = e / src.experts_per_peer, el = e % src.experts_per_peer;
    const __nv_bfloat16* row = reinterpret_cast<const __nv_bfloat16*>(src.ptr[peer]) +
                               ((size_t)el * G_total * C + (size_t)(g_off + g) * C + c) * M;
    const __nv_bfloat16* d = dout + (size_t)tok * M;
    for (int i = lane * 8; i < M; i += 256) {
      const int4 a = ld_nc_v4(d + i);
      const int4 b = *reinterpret_cast<const int4*>(row + i);
      const uint32_t* au = reinterpret_cast<const uint32_t*>(&a);
      const uint32_t* bu = reinterpret_cast<const uint32_t*>(&b);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fa = unpack_bf16x2(au[j]), fb = unpack_bf16x2(bu[j]);
        acc += fa.x * fb.x + fa.y * fb.y;
      }
    }
  }
  acc = warp_sum_f(acc);
  if (lane == 0) dw[wid] = __float2bfloat16(acc);
}

}  // namespace
}  // namespace ab

using namespace ab;

extern "C" int ab_moe_top2_route(const float* gates, int64_t* expert, int64_t* slot, int G, int S, int E, int C,
                                 cudaStream_t st) {
  if (E > kMaxExperts || E < 2) return 1;
  moe_top2_route_kernel<<<G, kRouteThreads, 0, st>>>(gates, expert, slot, S, E, C);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_moe_dispatch(const __nv_bfloat16* x, const int64_t* expert, const int64_t* slot,
                               const __nv_bfloat16* weight, const MoePeers* dst, int G, int S, int K, int M, int C,
                               int g_off, int G_total, cudaStream_t st) {
  if (M % 8) return 1;
  const long long warps = (long long)G * S * K;
  const int grid = (int)((warps + 7) / 8);
  moe_dispatch_kernel<<<grid, 256, 0, st>>>(x, expert, slot, weight, *dst, G * S, S, K, M, C, g_off, G_total);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_moe_combine(const MoePeers* src, const int64_t* expert, const int64_t* slot,
                              const __nv_bfloat16* weight, __nv_bfloat16* out, int G, int S, int K, int M, int C,
                              int g_off, int G_total, cudaStream_t st) {
  if (M % 8) return 1;
  const long long warps = (long long)G * S;
  const int grid = (int)((warps + 7) / 8);
  moe_combine_kernel<<<grid, 256, 0, st>>>(*src, expert, slot, weight, out, G * S, S, K, M, C, g_off, G_total);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_moe_combine_wgrad(const __nv_bfloat16* dout, const MoePeers* src, const int64_t* expert,
                                    const int64_t* slot, __nv_bfloat16* dw, int G, int S, int K, int M, int C,
                                    int g_off, int G_total, cudaStream_t st) {
  if (M % 8) return 1;
  const long long warps = (long long)G * S * K;
  const int grid = (int)((warps + 7) / 8);
  moe_combine_wgrad_kernel<<<grid, 256, 0, st>>>(dout, *src, expert, slot, dw, G * S, S, K, M, C, g_off, G_total);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
