// Bandwidth-bound sm_90a kernels: LayerNorm fwd/bwd (fused residual add), vocab-parallel softmax
// cross-entropy (stats + in-place gradient), embedding gather / scatter-add, column sum (bias grad),
// fused multi-tensor AdamW on fp32 master weights, grad-norm, bf16<->fp32 casts.
//
// Reference behaviour: XLA LLVM fusions for K6 (LayerNorm), K7/K8 (embedding as one-hot matmul and
// one-hot cross entropy, alpa/monkey_patch.py:241-247, benchmark_one_case_gpt_bert.py:114-118) and
// K9 (optimizer on fp32 master, alpa/model/model_util.py:282-327).  Here each is one pass over HBM
// with 128-bit accesses.
#include "kernels.h"
#include "ptx.cuh"

namespace ab {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int kThreads>
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (l < kThreads / 32) ? sh[l] : 0.f;
  return warp_sum(t);
}
template <int kThreads>
__device__ __forceinline__ float block_max(float v, float* sh) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (l < kThreads / 32) ? sh[l] : -INFINITY;
  return warp_max(t);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm.  One CTA per row (grid-stride), 8 bf16 per 128-bit access, row kept in registers.
// kRms: RMSNorm, the same kernels without the mean and beta: y = x * rstd * g, rstd = rsqrt(mean(x^2) + eps).
// ------------------------------------------------------------------------------------------------
constexpr int kLnThreads = 256;
constexpr int kLnMaxChunks = 8;  // H <= 256 * 8 * 8 = 16384

template <int kChunks, bool kRms>
__global__ void __launch_bounds__(kLnThreads)
layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                     const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
                     __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ sum_out,
                     float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int H,
                     float eps) {
  __shared__ float sh[32];
  const int nvec = H / 8;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    float v[kChunks][8];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const int vi = threadIdx.x + c * kLnThreads;
      if (vi < nvec) {
        int4 a = *reinterpret_cast<const int4*>(x + (size_t)row * H + vi * 8);
        const uint32_t* au = reinterpret_cast<const uint32_t*>(&a);
        if (res != nullptr) {
          int4 b = *reinterpret_cast<const int4*>(res + (size_t)row * H + vi * 8);
          const uint32_t* bu = reinterpret_cast<const uint32_t*>(&b);
          int4 o;
          uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 fa = unpack_bf16x2(au[j]), fb = unpack_bf16x2(bu[j]);
            ou[j] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
            float2 r = unpack_bf16x2(ou[j]);  // normalise the rounded sum (matches unfused path)
            v[c][2 * j] = r.x;
            v[c][2 * j + 1] = r.y;
          }
          if (sum_out != nullptr) *reinterpret_cast<int4*>(sum_out + (size_t)row * H + vi * 8) = o;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 fa = unpack_bf16x2(au[j]);
            v[c][2 * j] = fa.x;
            v[c][2 * j + 1] = fa.y;
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[c][j];
      }
    }
    float mean = 0.f;
    if constexpr (!kRms) mean = block_sum<kLnThreads>(s, sh) / H;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const int vi = threadIdx.x + c * kLnThreads;
      if (vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[c][j] - mean;
          q += d * d;
        }
      }
    }
    const float var = block_sum<kLnThreads>(q, sh) / H;
    const float rstd = rsqrtf(var + eps);
    if (threadIdx.x == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const int vi = threadIdx.x + c * kLnThreads;
      if (vi < nvec) {
        int4 g = *reinterpret_cast<const int4*>(gamma + vi * 8);
        const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
        int4 o;
        uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
        if constexpr (kRms) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 fg = unpack_bf16x2(gu[j]);
            ou[j] = pack_bf16x2(v[c][2 * j] * rstd * fg.x, v[c][2 * j + 1] * rstd * fg.y);
          }
        } else {
          int4 b = *reinterpret_cast<const int4*>(beta + vi * 8);
          const uint32_t* bu = reinterpret_cast<const uint32_t*>(&b);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 fg = unpack_bf16x2(gu[j]), fb = unpack_bf16x2(bu[j]);
            ou[j] = pack_bf16x2((v[c][2 * j] - mean) * rstd * fg.x + fb.x,
                                (v[c][2 * j + 1] - mean) * rstd * fg.y + fb.y);
          }
        }
        *reinterpret_cast<int4*>(y + (size_t)row * H + vi * 8) = o;
      }
    }
  }
}

// dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)) [+ dres];  dgamma += dy*xhat; dbeta += dy
// kRms: xhat = x * rstd, no mean(g*dy) term and no dbeta; the per-CTA slots hold dgamma only ([H] instead of [2][H]).
template <int kChunks, bool kRms>
__global__ void __launch_bounds__(kLnThreads)
layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                     const __nv_bfloat16* __restrict__ gamma, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dres,
                     __nv_bfloat16* __restrict__ dx, float* __restrict__ ws, int rows, int H) {
  __shared__ float sh[32];
  const int nvec = H / 8;
  float ag[kChunks][8], abt[kChunks][8];
#pragma unroll
  for (int c = 0; c < kChunks; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[c][j] = abt[c][j] = 0.f;

  constexpr int kParts = kRms ? 1 : 2;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const float mu = kRms ? 0.f : mean[row], rs = rstd[row];
    float xh[kChunks][8], gd[kChunks][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const int vi = threadIdx.x + c * kLnThreads;
      if (vi < nvec) {
        int4 a = *reinterpret_cast<const int4*>(x + (size_t)row * H + vi * 8);
        int4 d = *reinterpret_cast<const int4*>(dy + (size_t)row * H + vi * 8);
        int4 g = *reinterpret_cast<const int4*>(gamma + vi * 8);
        const uint32_t* au = reinterpret_cast<const uint32_t*>(&a);
        const uint32_t* du = reinterpret_cast<const uint32_t*>(&d);
        const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 fx = unpack_bf16x2(au[j]), fd = unpack_bf16x2(du[j]), fg = unpack_bf16x2(gu[j]);
          xh[c][2 * j] = (fx.x - mu) * rs;
          xh[c][2 * j + 1] = (fx.y - mu) * rs;
          gd[c][2 * j] = fd.x * fg.x;
          gd[c][2 * j + 1] = fd.y * fg.y;
          ag[c][2 * j] += fd.x * xh[c][2 * j];
          ag[c][2 * j + 1] += fd.y * xh[c][2 * j + 1];
          abt[c][2 * j] += fd.x;
          abt[c][2 * j + 1] += fd.y;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s1 += gd[c][j];
          s2 += gd[c][j] * xh[c][j];
        }
      }
    }
    float m1 = 0.f;
    if constexpr (!kRms) m1 = block_sum<kLnThreads>(s1, sh) / H;
    const float m2 = block_sum<kLnThreads>(s2, sh) / H;
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      const int vi = threadIdx.x + c * kLnThreads;
      if (vi < nvec) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (gd[c][j] - m1 - xh[c][j] * m2);
        if (dres != nullptr) {
          int4 r = *reinterpret_cast<const int4*>(dres + (size_t)row * H + vi * 8);
          const uint32_t* ru = reinterpret_cast<const uint32_t*>(&r);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float2 fr = unpack_bf16x2(ru[j]);
            o[2 * j] += fr.x;
            o[2 * j + 1] += fr.y;
          }
        }
        int4 ov;
        ov.x = pack_bf16x2(o[0], o[1]);
        ov.y = pack_bf16x2(o[2], o[3]);
        ov.z = pack_bf16x2(o[4], o[5]);
        ov.w = pack_bf16x2(o[6], o[7]);
        *reinterpret_cast<int4*>(dx + (size_t)row * H + vi * 8) = ov;
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kChunks; ++c) {
    const int vi = threadIdx.x + c * kLnThreads;
    if (vi < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {  // this CTA's partial sums (reduced in a fixed order by reduce_slots_kernel)
        ws[(size_t)blockIdx.x * kParts * H + vi * 8 + j] = ag[c][j];
        if constexpr (!kRms) ws[(size_t)blockIdx.x * 2 * H + H + vi * 8 + j] = abt[c][j];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Warp-group-per-row LayerNorm (H % (256*WPR) == 0): WPR warps share a row, VPL 128-bit loads in
// flight per lane, no CTA-wide barriers (row groups synchronise on their own named barrier).
// ------------------------------------------------------------------------------------------------
template <int WPR>
__device__ __forceinline__ void group_sum2(float& a, float& b, float2 (*xch)[WPR], int grp, int wr, int lane,
                                           int parity) {
  a = warp_sum(a);
  b = warp_sum(b);
  if constexpr (WPR > 1) {
    float2* slot = xch[(parity & 1) * 8 + grp];
    if (lane == 0) slot[wr] = make_float2(a, b);
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(32 * WPR) : "memory");
    a = 0.f;
    b = 0.f;
#pragma unroll
    for (int i = 0; i < WPR; ++i) {
      a += slot[i].x;
      b += slot[i].y;
    }
  }
}

// RMS: two CTAs per SM, else ptxas caps VPL = 8 at 80 registers and spills; 0 (no minimum) keeps LayerNorm's code.
template <int VPL, int WPR, bool kRms>
__global__ void __launch_bounds__(256, kRms ? 2 : 0)
layernorm_fwd_warp_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res,
                          const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
                          __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ sum_out,
                          float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, float eps) {
  constexpr int H = VPL * WPR * 256;
  __shared__ float2 xch[16][WPR];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int grp = wib / WPR, wr = wib % WPR;
  const int groups_per_cta = (blockDim.x >> 5) / WPR;
  const int ngroups = gridDim.x * groups_per_cta;
  int it = 0;
  for (int row = blockIdx.x * groups_per_cta + grp; row < rows; row += ngroups, ++it) {
    int4 v[VPL];
    const __nv_bfloat16* xr = x + (size_t)row * H;
#pragma unroll
    for (int c = 0; c < VPL; ++c) v[c] = ld_nc_v4(xr + ((c * WPR + wr) * 32 + lane) * 8);
    if (res != nullptr) {
      const __nv_bfloat16* rr = res + (size_t)row * H;
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const int off = ((c * WPR + wr) * 32 + lane) * 8;
        const int4 r = ld_nc_v4(rr + off);
        uint32_t* a = reinterpret_cast<uint32_t*>(&v[c]);
        const uint32_t* b = reinterpret_cast<const uint32_t*>(&r);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 fa = unpack_bf16x2(a[j]), fb = unpack_bf16x2(b[j]);
          a[j] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
        }
        if (sum_out != nullptr) *reinterpret_cast<int4*>(sum_out + (size_t)row * H + off) = v[c];
      }
    }
    float s = 0.f, dummy = 0.f, mean = 0.f;
    if constexpr (!kRms) {
#pragma unroll
      for (int c = 0; c < VPL; ++c) {
        const uint32_t* a = reinterpret_cast<const uint32_t*>(&v[c]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(a[j]);
          s += f.x + f.y;
        }
      }
      group_sum2<WPR>(s, dummy, xch, grp, wr, lane, 2 * it);
      mean = s * (1.f / H);
    }
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const uint32_t* a = reinterpret_cast<const uint32_t*>(&v[c]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(a[j]);
        q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
      }
    }
    // the exchange buffer must alternate between consecutive group sums (a fast warp may start the next one before a
    // slow warp has read this one's slots): LayerNorm makes two per row, RMSNorm only this one
    group_sum2<WPR>(q, dummy, xch, grp, wr, lane, kRms ? it : 2 * it + 1);
    const float rstd = rsqrtf(q * (1.f / H) + eps);
    if (lane == 0 && wr == 0) {
      if (mean_out) mean_out[row] = mean;
      if (rstd_out) rstd_out[row] = rstd;
    }
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int off = ((c * WPR + wr) * 32 + lane) * 8;
      const int4 g = *reinterpret_cast<const int4*>(gamma + off);
      const uint32_t* a = reinterpret_cast<const uint32_t*>(&v[c]);
      const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
      int4 o;
      uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
      if constexpr (kRms) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(a[j]), fg = unpack_bf16x2(gu[j]);
          ou[j] = pack_bf16x2(f.x * rstd * fg.x, f.y * rstd * fg.y);
        }
      } else {
        const int4 b = *reinterpret_cast<const int4*>(beta + off);
        const uint32_t* bu = reinterpret_cast<const uint32_t*>(&b);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(a[j]), fg = unpack_bf16x2(gu[j]), fb = unpack_bf16x2(bu[j]);
          ou[j] = pack_bf16x2((f.x - mean) * rstd * fg.x + fb.x, (f.y - mean) * rstd * fg.y + fb.y);
        }
      }
      *reinterpret_cast<int4*>(y + (size_t)row * H + off) = o;
    }
  }
}

template <int VPL, int WPR, bool kRms>
__global__ void __launch_bounds__(256)
layernorm_bwd_warp_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                          const __nv_bfloat16* __restrict__ gamma, const float* __restrict__ mean,
                          const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dres,
                          __nv_bfloat16* __restrict__ dx, float* __restrict__ ws, int rows) {
  constexpr int H = VPL * WPR * 256;
  constexpr int kParts = kRms ? 1 : 2;
  extern __shared__ float sh_gb[];   // [row groups][kParts][H]
  __shared__ float2 xch[16][WPR];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int grp = wib / WPR, wr = wib % WPR;
  const int groups_per_cta = (blockDim.x >> 5) / WPR;
  const int ngroups = gridDim.x * groups_per_cta;
  float ag[VPL][8], ab[VPL][8];
#pragma unroll
  for (int c = 0; c < VPL; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[c][j] = ab[c][j] = 0.f;
  int it = 0;
  for (int row = blockIdx.x * groups_per_cta + grp; row < rows; row += ngroups, ++it) {
    const float mu = kRms ? 0.f : mean[row], rs = rstd[row];
    int4 xv[VPL], dv[VPL];
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int off = ((c * WPR + wr) * 32 + lane) * 8;
      xv[c] = ld_nc_v4(x + (size_t)row * H + off);
      dv[c] = ld_nc_v4(dy + (size_t)row * H + off);
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int4 g = *reinterpret_cast<const int4*>(gamma + ((c * WPR + wr) * 32 + lane) * 8);
      const uint32_t* xu = reinterpret_cast<const uint32_t*>(&xv[c]);
      const uint32_t* du = reinterpret_cast<const uint32_t*>(&dv[c]);
      const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fx = unpack_bf16x2(xu[j]), fd = unpack_bf16x2(du[j]), fg = unpack_bf16x2(gu[j]);
        const float xh0 = (fx.x - mu) * rs, xh1 = (fx.y - mu) * rs;
        const float gd0 = fd.x * fg.x, gd1 = fd.y * fg.y;
        ag[c][2 * j] += fd.x * xh0;
        ag[c][2 * j + 1] += fd.y * xh1;
        ab[c][2 * j] += fd.x;
        ab[c][2 * j + 1] += fd.y;
        s1 += gd0 + gd1;
        s2 += gd0 * xh0 + gd1 * xh1;
      }
    }
    group_sum2<WPR>(s1, s2, xch, grp, wr, lane, it);
    const float m1 = kRms ? 0.f : s1 * (1.f / H), m2 = s2 * (1.f / H);
#pragma unroll
    for (int c = 0; c < VPL; ++c) {
      const int off = ((c * WPR + wr) * 32 + lane) * 8;
      const int4 g = *reinterpret_cast<const int4*>(gamma + off);
      const uint32_t* xu = reinterpret_cast<const uint32_t*>(&xv[c]);
      const uint32_t* du = reinterpret_cast<const uint32_t*>(&dv[c]);
      const uint32_t* gu = reinterpret_cast<const uint32_t*>(&g);
      int4 r = make_int4(0, 0, 0, 0);
      if (dres != nullptr) r = ld_nc_v4(dres + (size_t)row * H + off);
      const uint32_t* ru = reinterpret_cast<const uint32_t*>(&r);
      int4 o;
      uint32_t* ou = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fx = unpack_bf16x2(xu[j]), fd = unpack_bf16x2(du[j]), fg = unpack_bf16x2(gu[j]);
        const float2 fr = unpack_bf16x2(ru[j]);
        const float xh0 = (fx.x - mu) * rs, xh1 = (fx.y - mu) * rs;
        ou[j] = pack_bf16x2(rs * (fd.x * fg.x - m1 - xh0 * m2) + fr.x, rs * (fd.y * fg.y - m1 - xh1 * m2) + fr.y);
      }
      *reinterpret_cast<int4*>(dx + (size_t)row * H + off) = o;
    }
  }
  // CTA-level reduction of the per-lane partials in a fixed order (row group 0, 1, ...): every column has exactly one
  // owner lane per row group; the CTA's sums go to ws[blockIdx.x] and are reduced over CTAs by reduce_slots_kernel
#pragma unroll
  for (int c = 0; c < VPL; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = ((c * WPR + wr) * 32 + lane) * 8 + j;
      sh_gb[grp * kParts * H + col] = ag[c][j];
      if constexpr (!kRms) sh_gb[grp * 2 * H + H + col] = ab[c][j];
    }
  __syncthreads();
  for (int i = threadIdx.x; i < kParts * H; i += blockDim.x) {
    float t = 0.f;
    for (int g = 0; g < groups_per_cta; ++g) t += sh_gb[g * kParts * H + i];
    ws[(size_t)blockIdx.x * kParts * H + i] = t;
  }
}

// out[c] += sum over s = 0, 1, ... of ws[s * ld + c]: the fixed-order second pass of every cross-CTA reduction below,
// so results do not depend on which CTA finishes first.
__global__ void __launch_bounds__(256)
reduce_slots_kernel(const float* __restrict__ ws, int slots, long long ld, int n, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  float t = 0.f;
  for (int s = 0; s < slots; ++s) t += ws[(size_t)s * ld + c];
  out[c] += t;
}

// ------------------------------------------------------------------------------------------------
// Vocab-parallel cross entropy.  Pass 1: per-row (max, sum exp(x-max), target logit) over the local
// vocab shard.  (The tiny [rows,3] stats tensor is combined across the tensor-parallel group by the
// caller.)  Pass 2: logits <- (softmax - onehot) * scale in place, loss per row.
// ------------------------------------------------------------------------------------------------
constexpr int kCeThreads = 512;

__global__ void __launch_bounds__(kCeThreads)
ce_stats_kernel(const __nv_bfloat16* __restrict__ logits, const int64_t* __restrict__ labels,
                float* __restrict__ stats, int rows, int V, int vocab_start, long long ld) {
  __shared__ float sh[32];
  const int row = blockIdx.x;
  if (row >= rows) return;
  const __nv_bfloat16* p = logits + (size_t)row * ld;
  const int nvec = V / 8;
  float mx = -INFINITY;
  for (int vi = threadIdx.x; vi < nvec; vi += kCeThreads) {
    int4 a = *reinterpret_cast<const int4*>(p + vi * 8);
    const uint32_t* au = reinterpret_cast<const uint32_t*>(&a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = unpack_bf16x2(au[j]);
      mx = fmaxf(mx, fmaxf(f.x, f.y));
    }
  }
  mx = block_max<kCeThreads>(mx, sh);
  float se = 0.f;
  for (int vi = threadIdx.x; vi < nvec; vi += kCeThreads) {
    int4 a = *reinterpret_cast<const int4*>(p + vi * 8);
    const uint32_t* au = reinterpret_cast<const uint32_t*>(&a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = unpack_bf16x2(au[j]);
      se += __expf(f.x - mx) + __expf(f.y - mx);
    }
  }
  se = block_sum<kCeThreads>(se, sh);
  if (threadIdx.x == 0) {
    const long long lab = labels[row] - vocab_start;
    stats[row * 3 + 0] = mx;
    stats[row * 3 + 1] = se;
    stats[row * 3 + 2] = (lab >= 0 && lab < V) ? __bfloat162float(p[lab]) : 0.f;
  }
}

// gstats: [rows,2] = (global max, global sum exp relative to global max), tgt: global target logit.
__global__ void __launch_bounds__(kCeThreads)
ce_grad_kernel(__nv_bfloat16* __restrict__ logits, const int64_t* __restrict__ labels,
               const float* __restrict__ gstats, const float* __restrict__ row_scale,
               int rows, int V, int vocab_start, long long ld) {
  const int row = blockIdx.x;
  if (row >= rows) return;
  __nv_bfloat16* p = logits + (size_t)row * ld;
  const float mx = gstats[row * 2 + 0];
  const float inv = 1.f / gstats[row * 2 + 1];
  const float sc = row_scale[row];  // mask / num_valid * upstream grad
  const long long lab = labels[row] - vocab_start;
  const int nvec = V / 8;
  for (int vi = threadIdx.x; vi < nvec; vi += kCeThreads) {
    int4 a = *reinterpret_cast<const int4*>(p + vi * 8);
    uint32_t* au = reinterpret_cast<uint32_t*>(&a);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = unpack_bf16x2(au[j]);
      const int c = vi * 8 + 2 * j;
      float g0 = __expf(f.x - mx) * inv - (c == lab ? 1.f : 0.f);
      float g1 = __expf(f.y - mx) * inv - (c + 1 == lab ? 1.f : 0.f);
      au[j] = pack_bf16x2(g0 * sc, g1 * sc);
    }
    *reinterpret_cast<int4*>(p + vi * 8) = a;
  }
}

// ------------------------------------------------------------------------------------------------
// Embedding gather (+ position embedding) and scatter-add backward (fp32 main grads).
// Vocab-parallel: rows outside [vocab_start, vocab_start+Vlocal) produce zeros.
// ------------------------------------------------------------------------------------------------
__global__ void embedding_fwd_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos,
                                     const __nv_bfloat16* __restrict__ wte,
                                     const __nv_bfloat16* __restrict__ wpe,
                                     __nv_bfloat16* __restrict__ out, int T, int H, int vocab_start,
                                     int Vlocal) {
  const int nvec = H / 8;
  for (int t = blockIdx.x; t < T; t += gridDim.x) {
    const long long id = ids[t] - vocab_start;
    const bool ok = id >= 0 && id < Vlocal;
    for (int vi = threadIdx.x; vi < nvec; vi += blockDim.x) {
      int4 a = make_int4(0, 0, 0, 0);
      if (ok) a = *reinterpret_cast<const int4*>(wte + (size_t)id * H + vi * 8);
      if (wpe != nullptr) {
        int4 b = *reinterpret_cast<const int4*>(wpe + (size_t)pos[t] * H + vi * 8);
        uint32_t* au = reinterpret_cast<uint32_t*>(&a);
        const uint32_t* bu = reinterpret_cast<const uint32_t*>(&b);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 fa = unpack_bf16x2(au[j]), fb = unpack_bf16x2(bu[j]);
          au[j] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
        }
      }
      *reinterpret_cast<int4*>(out + (size_t)t * H + vi * 8) = a;
    }
  }
}

// sorted_ids / order: the token ids sorted stably and the token index of each sorted position.  The CTA at the first
// position of a run of equal ids sums that run's rows in token order and adds the result once: no atomics, so the
// gradient does not depend on scheduling.
__global__ void embedding_bwd_kernel(const int64_t* __restrict__ sorted_ids, const int64_t* __restrict__ order,
                                     const __nv_bfloat16* __restrict__ dy, float* __restrict__ dtable, int T, int H,
                                     int vocab_start, int Vlocal) {
  for (int i = blockIdx.x; i < T; i += gridDim.x) {
    const long long raw = sorted_ids[i];
    if (i > 0 && sorted_ids[i - 1] == raw) continue;
    const long long id = raw - vocab_start;
    if (id < 0 || id >= Vlocal) continue;
    int end = i + 1;
    while (end < T && sorted_ids[end] == raw) ++end;
    for (int c = threadIdx.x; c < H / 2; c += blockDim.x) {
      float sx = 0.f, sy = 0.f;
      for (int j = i; j < end; ++j) {
        const float2 f = unpack_bf16x2(reinterpret_cast<const uint32_t*>(dy + (size_t)order[j] * H)[c]);
        sx += f.x;
        sy += f.y;
      }
      float2* o = reinterpret_cast<float2*>(dtable + (size_t)id * H) + c;
      const float2 old = *o;
      *o = make_float2(old.x + sx, old.y + sy);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Column sum: out[n] (+)= sum_m x[m, n]   (bias gradients).  fp32 accumulate.
// ------------------------------------------------------------------------------------------------
// block = (32 column groups of 8) x (8 row lanes); 4 rows x 16 bytes in flight per thread
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ ws, int M, int N, long long ld,
              int rows_per_block) {
  __shared__ float red[8][256 + 8];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + tx) * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < N) {
    int r = r0 + ty;
    for (; r + 24 < r1; r += 32) {
      int4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld_nc_v4(x + (size_t)(r + 8 * u) * ld + col);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&v[u]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_bf16x2(w[j]);
          s[2 * j] += f.x;
          s[2 * j + 1] += f.y;
        }
      }
    }
    for (; r < r1; r += 8) {
      const int4 v = ld_nc_v4(x + (size_t)r * ld + col);
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(w[j]);
        s[2 * j] += f.x;
        s[2 * j + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[ty][tx * 8 + j] = s[j];
  __syncthreads();
  const int c = threadIdx.x;   // 256 columns per block
  if (blockIdx.x * 256 + c < N) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += red[y][c];
    ws[(size_t)blockIdx.y * N + blockIdx.x * 256 + c] = t;   // row block y's partial
  }
}

// ------------------------------------------------------------------------------------------------
// Fused multi-tensor AdamW.  Tensors are described by a device table; each CTA takes one chunk.
// grad fp32 (main grads) or bf16; master fp32; writes bf16 model weights.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adamw_kernel(const AdamTensor* __restrict__ tensors, const AdamChunk* __restrict__ chunks,
             int num_chunks, float lr, float beta1, float beta2, float eps, float bc1, float bc2,
             float grad_scale, const float* __restrict__ clip_coef, const float* __restrict__ step_ptr) {
  const float gs = grad_scale * (clip_coef != nullptr ? *clip_coef : 1.f);
  if (step_ptr != nullptr) {  // step count lives on the device (keeps the step graph-capturable)
    const float st = *step_ptr;
    bc1 = 1.f - powf(beta1, st);
    bc2 = 1.f - powf(beta2, st);
  }
  for (int ci = blockIdx.x; ci < num_chunks; ci += gridDim.x) {
    const AdamChunk ch = chunks[ci];
    const AdamTensor t = tensors[ch.tensor];
    const long long end = min(t.n, ch.start + (long long)kAdamChunk);
    for (long long i = ch.start + threadIdx.x * 4; i < end; i += 256 * 4) {
      float g[4], p[4], m[4], v[4];
      const bool full = i + 4 <= end;
      if (full) {
        if (t.grad_is_bf16) {
          const uint2 gv = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(t.grad) + i);
          float2 a = unpack_bf16x2(gv.x), b = unpack_bf16x2(gv.y);
          g[0] = a.x; g[1] = a.y; g[2] = b.x; g[3] = b.y;
        } else {
          const float4 gv = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(t.grad) + i);
          g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
        }
        const float4 pv = *reinterpret_cast<const float4*>(t.master + i);
        const float4 mv = *reinterpret_cast<const float4*>(t.m + i);
        const float4 vv = *reinterpret_cast<const float4*>(t.v + i);
        p[0] = pv.x; p[1] = pv.y; p[2] = pv.z; p[3] = pv.w;
        m[0] = mv.x; m[1] = mv.y; m[2] = mv.z; m[3] = mv.w;
        v[0] = vv.x; v[1] = vv.y; v[2] = vv.z; v[3] = vv.w;
      } else {
        for (int j = 0; j < 4; ++j) {
          const long long k = i + j;
          if (k < end) {
            g[j] = t.grad_is_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(t.grad)[k])
                                  : reinterpret_cast<const float*>(t.grad)[k];
            p[j] = t.master[k]; m[j] = t.m[k]; v[j] = t.v[k];
          } else {
            g[j] = p[j] = m[j] = v[j] = 0.f;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gg = g[j] * gs;
        m[j] = beta1 * m[j] + (1.f - beta1) * gg;
        v[j] = beta2 * v[j] + (1.f - beta2) * gg * gg;
        const float mh = m[j] / bc1, vh = v[j] / bc2;
        p[j] = p[j] - lr * (mh / (sqrtf(vh) + eps) + t.weight_decay * p[j]);
      }
      if (full) {
        *reinterpret_cast<float4*>(t.master + i) = make_float4(p[0], p[1], p[2], p[3]);
        *reinterpret_cast<float4*>(t.m + i) = make_float4(m[0], m[1], m[2], m[3]);
        *reinterpret_cast<float4*>(t.v + i) = make_float4(v[0], v[1], v[2], v[3]);
        if (t.param_bf16 != nullptr)
          *reinterpret_cast<uint2*>(t.param_bf16 + i) =
              make_uint2(pack_bf16x2(p[0], p[1]), pack_bf16x2(p[2], p[3]));
      } else {
        for (int j = 0; j < 4; ++j) {
          const long long k = i + j;
          if (k < end) {
            t.master[k] = p[j]; t.m[k] = m[j]; t.v[k] = v[j];
            if (t.param_bf16 != nullptr) t.param_bf16[k] = __float2bfloat16(p[j]);
          }
        }
      }
    }
  }
}

// sum of squares over a table of tensors -> out[0] (fp32), for global-norm clipping.
__global__ void __launch_bounds__(256)
sumsq_kernel(const AdamTensor* __restrict__ tensors, const AdamChunk* __restrict__ chunks,
             int num_chunks, float* __restrict__ ws) {
  __shared__ float sh[32];
  float s = 0.f;
  for (int ci = blockIdx.x; ci < num_chunks; ci += gridDim.x) {
    const AdamChunk ch = chunks[ci];
    const AdamTensor t = tensors[ch.tensor];
    const long long end = min(t.n, ch.start + (long long)kAdamChunk);
    for (long long i = ch.start + threadIdx.x; i < end; i += 256) {
      const float g = t.grad_is_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(t.grad)[i])
                                     : reinterpret_cast<const float*>(t.grad)[i];
      s += g * g;
    }
  }
  s = block_sum<256>(s, sh);
  if (threadIdx.x == 0) ws[blockIdx.x] = s;
}

}  // namespace ab

using namespace ab;

template <int kChunks, bool kRms>
static void ln_fwd_launch(const LayerNormArgs& a, cudaStream_t st, int grid) {
  layernorm_fwd_kernel<kChunks, kRms><<<grid, kLnThreads, 0, st>>>(
      a.x, a.residual, a.gamma, a.beta, a.y, a.sum_out, a.mean, a.rstd, a.rows, a.H, a.eps);
}
template <int kChunks, bool kRms>
static void ln_bwd_launch(const LayerNormBwdArgs& a, cudaStream_t st, int grid) {
  layernorm_bwd_kernel<kChunks, kRms><<<grid, kLnThreads, 0, st>>>(
      a.dy, a.x, a.gamma, a.mean, a.rstd, a.dres, a.dx, a.ws, a.rows, a.H);
}
static int ln_bwd_generic_grid(int rows) { return rows < ab::num_sms() * 2 ? rows : ab::num_sms() * 2; }
template <int WPR>
static int ln_bwd_warp_grid(int rows) {
  const int gpc = 8 / WPR;
  int grid = (rows + gpc - 1) / gpc;
  if (grid > ab::num_sms() * 2) {
    const int iters = (rows + ab::num_sms() * 2 * gpc - 1) / (ab::num_sms() * 2 * gpc);
    grid = (rows + iters * gpc - 1) / (iters * gpc);
  }
  return grid;
}

template <int VPL, int WPR, bool kRms>
static void ln_fwd_warp_launch(const LayerNormArgs& a, cudaStream_t st) {
  const int gpc = 8 / WPR;
  int grid = (a.rows + gpc - 1) / gpc;
  if (grid > ab::num_sms() * 8) {
    // balanced persistent grid: every row group runs the same number of rows (16384 rows on 1184 CTAs would leave a
    // 27 % idle tail: some groups get 2 rows, most of the second wave only 1)
    const int iters = (a.rows + ab::num_sms() * 8 * gpc - 1) / (ab::num_sms() * 8 * gpc);
    grid = (a.rows + iters * gpc - 1) / (iters * gpc);
  }
  layernorm_fwd_warp_kernel<VPL, WPR, kRms><<<grid, 256, 0, st>>>(a.x, a.residual, a.gamma, a.beta, a.y, a.sum_out,
                                                                  a.mean, a.rstd, a.rows, a.eps);
}
template <int VPL, int WPR, bool kRms>
static void ln_bwd_warp_launch(const LayerNormBwdArgs& a, cudaStream_t st) {
  const int gpc = 8 / WPR;
  constexpr int H = VPL * WPR * 256;
  const int grid = ln_bwd_warp_grid<WPR>(a.rows);
  const int smem = gpc * (kRms ? 1 : 2) * H * (int)sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(layernorm_bwd_warp_kernel<VPL, WPR, kRms>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr_set = true;
  }
  layernorm_bwd_warp_kernel<VPL, WPR, kRms><<<grid, 256, smem, st>>>(
      a.dy, a.x, a.gamma, a.mean, a.rstd, a.dres, a.dx, a.ws, a.rows);
}

template <bool kRms>
static void ln_fwd_dispatch(const LayerNormArgs* a, cudaStream_t st) {
  if (a->H % 256 == 0 && a->H <= 8192) {
    switch (a->H / 256) {
      case 1: ln_fwd_warp_launch<1, 1, kRms>(*a, st); return;
      case 2: ln_fwd_warp_launch<2, 1, kRms>(*a, st); return;
      case 3: ln_fwd_warp_launch<3, 1, kRms>(*a, st); return;
      case 4: ln_fwd_warp_launch<4, 1, kRms>(*a, st); return;
      case 6: ln_fwd_warp_launch<6, 1, kRms>(*a, st); return;
      case 8: ln_fwd_warp_launch<8, 1, kRms>(*a, st); return;
      case 10: ln_fwd_warp_launch<5, 2, kRms>(*a, st); return;
      case 12: ln_fwd_warp_launch<6, 2, kRms>(*a, st); return;
      case 16: ln_fwd_warp_launch<8, 2, kRms>(*a, st); return;
      case 20: ln_fwd_warp_launch<5, 4, kRms>(*a, st); return;
      case 24: ln_fwd_warp_launch<6, 4, kRms>(*a, st); return;
      case 28: ln_fwd_warp_launch<7, 4, kRms>(*a, st); return;
      case 32: ln_fwd_warp_launch<8, 4, kRms>(*a, st); return;
      default: break;
    }
  }
  const int chunks = (a->H / 8 + kLnThreads - 1) / kLnThreads;
  const int grid = a->rows < ab::num_sms() * 8 ? a->rows : ab::num_sms() * 8;
  if (chunks <= 1) ln_fwd_launch<1, kRms>(*a, st, grid);
  else if (chunks <= 2) ln_fwd_launch<2, kRms>(*a, st, grid);
  else if (chunks <= 4) ln_fwd_launch<4, kRms>(*a, st, grid);
  else ln_fwd_launch<8, kRms>(*a, st, grid);
}
extern "C" int ab_layernorm_fwd(const LayerNormArgs* a, cudaStream_t st) {
  if (a->H % 8 != 0 || a->H > kLnThreads * 8 * kLnMaxChunks) return 1;
  if (a->rms) ln_fwd_dispatch<true>(a, st);
  else ln_fwd_dispatch<false>(a, st);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
// (VPL, WPR) of the warp-group kernel for H, or 0 when the generic kernel runs
static int ln_bwd_warp_cfg(int H) {
  if (H % 256 != 0 || H > 8192) return 0;
  switch (H / 256) {
    case 1: return 11; case 2: return 21; case 3: return 31; case 4: return 41; case 6: return 32; case 8: return 42;
    case 10: return 52; case 12: return 34; case 16: return 44; case 20: return 54; case 24: return 38; case 32: return 48;
  }
  return 0;
}
// Number of per-CTA partial rows ([2][H] floats each, [H] for RMSNorm) ab_layernorm_bwd writes into a.ws.
extern "C" int ab_layernorm_bwd_slots(int rows, int H) {
  const int cfg = ln_bwd_warp_cfg(H);
  if (cfg == 0) return ln_bwd_generic_grid(rows);
  switch (cfg % 10) {
    case 1: return ln_bwd_warp_grid<1>(rows);
    case 2: return ln_bwd_warp_grid<2>(rows);
    case 4: return ln_bwd_warp_grid<4>(rows);
    default: return ln_bwd_warp_grid<8>(rows);
  }
}
template <bool kRms>
static void ln_bwd_dispatch(const LayerNormBwdArgs* a, cudaStream_t st) {
  switch (ln_bwd_warp_cfg(a->H)) {
    case 11: ln_bwd_warp_launch<1, 1, kRms>(*a, st); break;
    case 21: ln_bwd_warp_launch<2, 1, kRms>(*a, st); break;
    case 31: ln_bwd_warp_launch<3, 1, kRms>(*a, st); break;
    case 41: ln_bwd_warp_launch<4, 1, kRms>(*a, st); break;
    case 32: ln_bwd_warp_launch<3, 2, kRms>(*a, st); break;
    case 42: ln_bwd_warp_launch<4, 2, kRms>(*a, st); break;
    case 52: ln_bwd_warp_launch<5, 2, kRms>(*a, st); break;
    case 34: ln_bwd_warp_launch<3, 4, kRms>(*a, st); break;
    case 44: ln_bwd_warp_launch<4, 4, kRms>(*a, st); break;
    case 54: ln_bwd_warp_launch<5, 4, kRms>(*a, st); break;
    case 38: ln_bwd_warp_launch<3, 8, kRms>(*a, st); break;
    case 48: ln_bwd_warp_launch<4, 8, kRms>(*a, st); break;
    default: {
      const int chunks = (a->H / 8 + kLnThreads - 1) / kLnThreads;
      const int grid = ln_bwd_generic_grid(a->rows);
      if (chunks <= 1) ln_bwd_launch<1, kRms>(*a, st, grid);
      else if (chunks <= 2) ln_bwd_launch<2, kRms>(*a, st, grid);
      else ln_bwd_launch<4, kRms>(*a, st, grid);
    }
  }
}
extern "C" int ab_layernorm_bwd(const LayerNormBwdArgs* a, cudaStream_t st) {
  if (a->H % 8 != 0 || a->H > kLnThreads * 8 * 4 || a->ws == nullptr) return 1;
  if (a->rms) ln_bwd_dispatch<true>(a, st);
  else ln_bwd_dispatch<false>(a, st);
  const int slots = ab_layernorm_bwd_slots(a->rows, a->H);
  const int blocks = (a->H + 255) / 256;
  const long long ld = (a->rms ? 1LL : 2LL) * a->H;
  reduce_slots_kernel<<<blocks, 256, 0, st>>>(a->ws, slots, ld, a->H, a->dgamma);
  if (!a->rms) reduce_slots_kernel<<<blocks, 256, 0, st>>>(a->ws + a->H, slots, ld, a->H, a->dbeta);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
extern "C" int ab_ce_stats(const __nv_bfloat16* logits, const int64_t* labels, float* stats, int rows,
                           int V, int vocab_start, long long ld, cudaStream_t st) {
  if (V % 8 != 0 || ld % 8 != 0) return 1;
  ce_stats_kernel<<<rows, kCeThreads, 0, st>>>(logits, labels, stats, rows, V, vocab_start, ld);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
extern "C" int ab_ce_grad(__nv_bfloat16* logits, const int64_t* labels, const float* gstats,
                          const float* row_scale, int rows, int V, int vocab_start, long long ld,
                          cudaStream_t st) {
  if (V % 8 != 0 || ld % 8 != 0) return 1;
  ce_grad_kernel<<<rows, kCeThreads, 0, st>>>(logits, labels, gstats, row_scale, rows, V, vocab_start, ld);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
extern "C" int ab_embedding_fwd(const int64_t* ids, const int64_t* pos, const __nv_bfloat16* wte,
                                const __nv_bfloat16* wpe, __nv_bfloat16* out, int T, int H,
                                int vocab_start, int Vlocal, cudaStream_t st) {
  if (H % 8 != 0) return 1;
  const int grid = T < ab::num_sms() * 16 ? T : ab::num_sms() * 16;
  embedding_fwd_kernel<<<grid, 128, 0, st>>>(ids, pos, wte, wpe, out, T, H, vocab_start, Vlocal);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
extern "C" int ab_embedding_bwd(const int64_t* sorted_ids, const int64_t* order, const __nv_bfloat16* dy,
                                float* dtable, int T, int H, int vocab_start, int Vlocal, cudaStream_t st) {
  if (H % 2 != 0) return 1;
  const int grid = T < ab::num_sms() * 16 ? T : ab::num_sms() * 16;
  embedding_bwd_kernel<<<grid, 256, 0, st>>>(sorted_ids, order, dy, dtable, T, H, vocab_start, Vlocal);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
// row blocks of the column sum (partials written to ws[gy][N])
static int colsum_rows_per_block(int M, int N) {
  const int gx = (N + 255) / 256;
  int gy = (ab::num_sms() * 8 + gx - 1) / gx;
  if (gy > (M + 31) / 32) gy = (M + 31) / 32;
  if (gy < 1) gy = 1;
  return (M + gy - 1) / gy;
}
extern "C" int ab_colsum_slots(int M, int N) {
  const int rpb = colsum_rows_per_block(M, N);
  return (M + rpb - 1) / rpb;
}
extern "C" int ab_colsum(const __nv_bfloat16* x, float* out, float* ws, int M, int N, long long ld,
                         cudaStream_t st) {
  if (N % 8 != 0 || ld % 8 != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || M <= 0) return 1;
  const int gx = (N + 255) / 256;
  const int rpb = colsum_rows_per_block(M, N);
  const int gy = ab_colsum_slots(M, N);
  colsum_kernel<<<dim3(gx, gy), 256, 0, st>>>(x, ws, M, N, ld, rpb);
  reduce_slots_kernel<<<gx, 256, 0, st>>>(ws, gy, N, N, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
extern "C" int ab_adamw(const AdamTensor* tensors, const AdamChunk* chunks, int num_chunks, float lr,
                        float beta1, float beta2, float eps, float bc1, float bc2, float grad_scale,
                        const float* clip_coef, const float* step_ptr, cudaStream_t st) {
  if (num_chunks <= 0) return 0;
  const int grid = num_chunks < ab::num_sms() * 8 ? num_chunks : ab::num_sms() * 8;
  adamw_kernel<<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, lr, beta1, beta2, eps, bc1, bc2,
                                     grad_scale, clip_coef, step_ptr);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
extern "C" int ab_sumsq_slots(int num_chunks) { return num_chunks < ab::num_sms() * 4 ? num_chunks : ab::num_sms() * 4; }
extern "C" int ab_sumsq(const AdamTensor* tensors, const AdamChunk* chunks, int num_chunks, float* out, float* ws,
                        cudaStream_t st) {
  if (num_chunks <= 0) return 0;
  const int grid = ab_sumsq_slots(num_chunks);
  sumsq_kernel<<<grid, 256, 0, st>>>(tensors, chunks, num_chunks, ws);
  reduce_slots_kernel<<<1, 256, 0, st>>>(ws, grid, 1, 1, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}
