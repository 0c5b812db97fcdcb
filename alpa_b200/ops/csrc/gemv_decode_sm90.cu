// Weight-streaming GEMV for the decode step of LLM serving (K20 of SURVEY.md §2.5: OPT decode, fp8 weights).
//
//   y[m, n] = act( sum_k LN(x)[m, k] * W[n, k] * w_scale[n] + bias[n] ) (+ residual[m, n])        m <= 8 tokens
//
// A decode step multiplies one token (or a handful) by every weight matrix: the time is the time to stream the weights
// from HBM once.  The first version of this kernel de-quantised the weights on the CUDA cores (one warp per output
// channel): ~70 instructions per 16-byte load, measured 2.4 TB/s -- instruction bound, not memory bound.  This version
// feeds the streamed bytes to the tensor cores UNCONVERTED:
//   * a CTA owns 16 output channels; its 8 warps split K.  A lane loads 16 contiguous bytes of weight row g (= lane / 4)
//     and of row g + 8 at k = block * 64 + (lane % 4) * 16: two mma.sync.m16n8k32 (e4m3) -- or m16n8k16 (bf16), 32 k per
//     block -- consume them as the A fragment.  The k index inside a block is permuted relative to the instruction's
//     canonical order, which is harmless for a dot product as long as B uses the same permutation: lane (g, c) loads the
//     16 bytes of token g's activations at the same k offsets from shared memory.  Per 1 KB of weights a warp issues
//     2 global loads, 1 shared load and 2 MMAs.
//   * n = 8 columns of the MMA are the (up to 8) tokens of the step.
//   * fp8 weights: the activations are quantised per token to e4m3 in the prologue (same numerics as the prefill GEMM,
//     gemm_sm90.cu); bf16 weights: bf16 activations.  The optional layer norm (or RMSNorm, RMS = true) of x is fused
//     into the same prologue: every CTA normalises / quantises the <= 8 rows itself (a few KB from L2) into shared
//     memory.
//   * split-K partials are reduced through shared memory; scale / bias / GELU | ReLU / residual in the epilogue.
//   * the first weight loads are issued before the programmatic-dependent-launch wait (pdl.h).
// Reference behaviour: the decode path of examples/llm_serving/model/opt_model.py (XLA cuBLAS GEMMs on fp16 weights).
#include <cuda_fp8.h>

#include "kernels.h"
#include "pdl.h"
#include "ptx.cuh"

namespace ab {

constexpr int kGemvWarps = 8;
constexpr int kGemvThreads = kGemvWarps * 32;
constexpr int kGemvRows = 16;          // output channels per CTA (the M of the MMA)
constexpr int kGemvBatch = 5;          // k blocks whose loads are in flight together (10 x 16 bytes per lane)

__device__ __forceinline__ void mma_e4m3(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_bf16(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float block_sum(float v, float* red, int warp, int lane) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                 // red[] may still be read from the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kGemvWarps; ++w) t += red[w];
  return t;
}
__device__ __forceinline__ float block_max(float v, float* red, int warp, int lane) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kGemvWarps; ++w) t = fmaxf(t, red[w]);
  return t;
}

template <bool FP8, bool RMS>
__global__ void __launch_bounds__(kGemvThreads) gemv_decode_kernel(const GemvArgs a) {
  constexpr int kEs = FP8 ? 1 : 2;            // bytes per weight / staged activation
  constexpr int kBlk = 64 / kEs;              // k per block: 16 bytes per lane quarter
  extern __shared__ __align__(16) uint8_t gemv_smem[];
  __shared__ float red[kGemvWarps];
  __shared__ float xscale[8];
  __shared__ float part[kGemvWarps][kGemvRows][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, c = lane & 3;
  const int N = a.N, K = a.K, M = a.M;
  const int n0 = blockIdx.x * kGemvRows;
  const int blocks = K / kBlk;                // K is a multiple of the block (checked on the host)
  const int per = (blocks + kGemvWarps - 1) / kGemvWarps;
  const int b_begin = min(warp * per, blocks), b_end = min(b_begin + per, blocks);
  // rows beyond N read row N - 1 (their results are dropped)
  const uint8_t* w0 = reinterpret_cast<const uint8_t*>(a.w) + (size_t)min(n0 + g, N - 1) * K * kEs + c * 16;
  const uint8_t* w1 = reinterpret_cast<const uint8_t*>(a.w) + (size_t)min(n0 + g + 8, N - 1) * K * kEs + c * 16;

  int4 wa[kGemvBatch], wb[kGemvBatch];
  auto load_batch = [&](int b0) {
#pragma unroll
    for (int u = 0; u < kGemvBatch; ++u) {
      const int b = b0 + u;
      if (b < b_end) {
        wa[u] = ld_nc_v4(w0 + (size_t)b * 64);
        wb[u] = ld_nc_v4(w1 + (size_t)b * 64);
      }
    }
  };
  load_batch(b_begin);                        // weights do not depend on the previous kernel
  griddep_launch_dependents();
  griddep_wait();

  // ---- prologue: (layer norm ->) (per-token e4m3 quantisation ->) shared memory, one token row after the other ----
  uint8_t* xs = gemv_smem;                    // [M][K] e4m3 or bf16
  const bool ln = a.ln_gamma != nullptr;
  const int xchunks = K / 8;                  // 16-byte pieces of a bf16 row
  for (int m = 0; m < M; ++m) {
    const __nv_bfloat16* xrow = a.x + (size_t)m * a.ldx;
    float mean = 0.f, rstd = 1.f;
    if (RMS) {
      // one pass: RMSNorm has no mean to subtract
      float s2 = 0.f;
      for (int i = threadIdx.x; i < xchunks; i += kGemvThreads) {
        const int4 v = *reinterpret_cast<const int4*>(xrow + (size_t)i * 8);
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = unpack_bf16x2(u[q]);
          s2 = fmaf(f.x, f.x, fmaf(f.y, f.y, s2));
        }
      }
      rstd = rsqrtf(block_sum(s2, red, warp, lane) / (float)K + a.ln_eps);
    } else if (ln) {
      // two passes over the row (it stays in L1 / L2), like the stand-alone layer norm: s2/K - mean^2 cancels
      // catastrophically in fp32 when |mean| >> std
      float s1 = 0.f, s2 = 0.f;
      for (int i = threadIdx.x; i < xchunks; i += kGemvThreads) {
        const int4 v = *reinterpret_cast<const int4*>(xrow + (size_t)i * 8);
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = unpack_bf16x2(u[q]);
          s1 += f.x + f.y;
        }
      }
      mean = block_sum(s1, red, warp, lane) / (float)K;
      for (int i = threadIdx.x; i < xchunks; i += kGemvThreads) {
        const int4 v = *reinterpret_cast<const int4*>(xrow + (size_t)i * 8);
        const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 f = unpack_bf16x2(u[q]);
          const float dx = f.x - mean, dy = f.y - mean;
          s2 = fmaf(dx, dx, fmaf(dy, dy, s2));
        }
      }
      rstd = rsqrtf(block_sum(s2, red, warp, lane) / (float)K + a.ln_eps);
    }
    auto value8 = [&](int i, float* f) {      // 8 (normalised, bf16-rounded) activations of chunk i
      const int4 v = *reinterpret_cast<const int4*>(xrow + (size_t)i * 8);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
      if (RMS) {
        const int4 gv = *reinterpret_cast<const int4*>(a.ln_gamma + (size_t)i * 8);
        const uint32_t* gu = reinterpret_cast<const uint32_t*>(&gv);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 x2 = unpack_bf16x2(u[q]), g2 = unpack_bf16x2(gu[q]);
          // round to bf16 like the stand-alone RMSNorm kernel does
          const float2 r = unpack_bf16x2(pack_bf16x2(x2.x * rstd * g2.x, x2.y * rstd * g2.y));
          f[2 * q] = r.x;
          f[2 * q + 1] = r.y;
        }
      } else if (ln) {
        const int4 gv = *reinterpret_cast<const int4*>(a.ln_gamma + (size_t)i * 8);
        const int4 bv = *reinterpret_cast<const int4*>(a.ln_beta + (size_t)i * 8);
        const uint32_t* gu = reinterpret_cast<const uint32_t*>(&gv);
        const uint32_t* bu = reinterpret_cast<const uint32_t*>(&bv);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 x2 = unpack_bf16x2(u[q]), g2 = unpack_bf16x2(gu[q]), b2 = unpack_bf16x2(bu[q]);
          // round to bf16 like the stand-alone layer norm kernel does
          const float2 r = unpack_bf16x2(pack_bf16x2(fmaf((x2.x - mean) * rstd, g2.x, b2.x),
                                                     fmaf((x2.y - mean) * rstd, g2.y, b2.y)));
          f[2 * q] = r.x;
          f[2 * q + 1] = r.y;
        }
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 x2 = unpack_bf16x2(u[q]);
          f[2 * q] = x2.x;
          f[2 * q + 1] = x2.y;
        }
      }
    };
    if (FP8) {
      float amax = 0.f;
      for (int i = threadIdx.x; i < xchunks; i += kGemvThreads) {
        float f[8];
        value8(i, f);
#pragma unroll
        for (int q = 0; q < 8; ++q) amax = fmaxf(amax, fabsf(f[q]));
      }
      amax = block_max(amax, red, warp, lane);
      const float sc = fmaxf(amax, 1e-8f) * (1.f / 448.f);   // quantize_rows_e4m3_kernel's formula, bit for bit
      const float inv = 1.f / sc;
      if (threadIdx.x == 0) xscale[m] = sc;
      for (int i = threadIdx.x; i < xchunks; i += kGemvThreads) {
        float f[8];
        value8(i, f);
        uint32_t o[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const __nv_fp8x4_e4m3 p(make_float4(f[4 * q] * inv, f[4 * q + 1] * inv, f[4 * q + 2] * inv, f[4 * q + 3] * inv));
          o[q] = *reinterpret_cast<const uint32_t*>(&p);
        }
        *reinterpret_cast<uint2*>(xs + (size_t)m * K + (size_t)i * 8) = make_uint2(o[0], o[1]);
      }
    } else {
      if (threadIdx.x == 0) xscale[m] = 1.f;
      for (int i = threadIdx.x; i < xchunks; i += kGemvThreads) {
        float f[8];
        value8(i, f);
        int4 o;
        o.x = pack_bf16x2(f[0], f[1]);
        o.y = pack_bf16x2(f[2], f[3]);
        o.z = pack_bf16x2(f[4], f[5]);
        o.w = pack_bf16x2(f[6], f[7]);
        *reinterpret_cast<int4*>(xs + ((size_t)m * K + (size_t)i * 8) * 2) = o;
      }
    }
  }
  __syncthreads();

  // ---- main loop: this warp's k blocks, kGemvBatch at a time ----
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const uint8_t* xq = xs + (size_t)g * K * kEs + c * 16;      // token g (only read when g < M)
  for (int b0 = b_begin; b0 < b_end; b0 += kGemvBatch) {
    if (b0 != b_begin) load_batch(b0);
#pragma unroll
    for (int u = 0; u < kGemvBatch; ++u) {
      const int b = b0 + u;
      if (b >= b_end) break;
      int4 xv = make_int4(0, 0, 0, 0);
      if (g < M) xv = *reinterpret_cast<const int4*>(xq + (size_t)b * 64);
      const uint32_t* pa = reinterpret_cast<const uint32_t*>(&wa[u]);
      const uint32_t* pb = reinterpret_cast<const uint32_t*>(&wb[u]);
      const uint32_t f0[4] = {pa[0], pb[0], pa[1], pb[1]};
      const uint32_t f1[4] = {pa[2], pb[2], pa[3], pb[3]};
      if (FP8) {
        mma_e4m3(acc, f0, (uint32_t)xv.x, (uint32_t)xv.y);
        mma_e4m3(acc, f1, (uint32_t)xv.z, (uint32_t)xv.w);
      } else {
        mma_bf16(acc, f0, (uint32_t)xv.x, (uint32_t)xv.y);
        mma_bf16(acc, f1, (uint32_t)xv.z, (uint32_t)xv.w);
      }
    }
  }
  // C fragment: acc[0], acc[1] = (row g, tokens 2c, 2c + 1); acc[2], acc[3] = (row g + 8, same tokens)
  part[warp][g][2 * c] = acc[0];
  part[warp][g][2 * c + 1] = acc[1];
  part[warp][g + 8][2 * c] = acc[2];
  part[warp][g + 8][2 * c + 1] = acc[3];
  __syncthreads();
  if (threadIdx.x < kGemvRows * 8) {
    const int r = threadIdx.x >> 3, m = threadIdx.x & 7;
    const int n = n0 + r;
    if (m < M && n < N) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kGemvWarps; ++w) v += part[w][r][m];
      v *= xscale[m] * (a.w_scale != nullptr ? a.w_scale[n] : 1.f);
      if (a.bias != nullptr) v += __bfloat162float(a.bias[n]);
      if (a.act == 1) v = 0.5f * v * (1.f + erff(v * 0.7071067811865476f));
      else if (a.act == 2) v = fmaxf(v, 0.f);
      if (a.residual != nullptr) v += __bfloat162float(a.residual[(size_t)m * a.ldr + n]);
      a.y[(size_t)m * a.ldy + n] = __float2bfloat16(v);
    }
  }
}

template <bool FP8, bool RMS>
static int gemv_launch(const GemvArgs& a, cudaStream_t st) {
  const int grid = (a.N + kGemvRows - 1) / kGemvRows;
  const size_t smem = (size_t)a.M * a.K * (FP8 ? 1 : 2);
  auto kern = gemv_decode_kernel<FP8, RMS>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return 100 + (int)e;
  }
  const cudaError_t e = launch_pdl(kern, dim3(grid), dim3(kGemvThreads), smem, st, a);
  return e == cudaSuccess ? 0 : 100 + (int)e;
}

}  // namespace ab

extern "C" int ab_gemv_decode(const ab::GemvArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->M < 1 || a->M > 8 || a->N <= 0) return 1;
  if (a->K % (a->fp8 ? 64 : 32) != 0 || a->ldx % 8 != 0) return 1;
  if ((size_t)a->M * a->K * (a->fp8 ? 1 : 2) > 200 * 1024) return 3;      // staged activations must fit shared memory
  if (a->ln_rms) {
    if (a->ln_gamma == nullptr || a->ln_beta != nullptr) return 3;
    return a->fp8 ? gemv_launch<true, true>(*a, st) : gemv_launch<false, true>(*a, st);
  }
  if (a->ln_gamma != nullptr && a->ln_beta == nullptr) return 3;
  return a->fp8 ? gemv_launch<true, false>(*a, st) : gemv_launch<false, false>(*a, st);
}
