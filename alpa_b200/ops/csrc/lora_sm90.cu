// Multi-LoRA shrink and expand over the segments of a ragged token batch (serving many adapters over one base model).
//
//   shrink:  y[p, i, :] = sum over split p's K range of  x[rows[i], k] * A[slot][:, k]          fp32 partials
//   expand:  out[rows[i], :] = bf16(float(out[rows[i], :]) + scale[slot] * (sum_p y[p, i, :]) . B[slot]^T)   in place
//
// The host sorts the tokens that carry an adapter by adapter slot: `rows` [Tl] are their batch rows, segment s is
// rows[seg_start[s] .. seg_start[s + 1]) and uses slot seg_slot[s].  A row of `out` that no segment lists is never
// read or written.  A: [slots, R, K], B: [slots, N, R] bf16, scale: [slots] fp32.
//
// * Tiles.  A CTA (4 warps) serves BM = 16 * MT rows of one segment; tiles are numbered segment by segment and the grid
//   is an upper bound (ceil(Tl / BM) + S tiles), so no descriptor is read on the host.  MT = 1 when segments are decode
//   sized (a few rows), 4 for prefill segments.
// * Tensor cores: mma.sync m16n8k16 bf16, fp32 accumulation.  A lane loads 16 contiguous bytes of a row at
//   k = k0 + 8 * (lane % 4) for both operands and feeds them to two MMAs: the k order inside a 32-wide step is permuted
//   the same way for both operands, which a dot product does not see (as in gemv_decode_sm90.cu).
// * Shrink: the warps split R (n8 tiles w, w + 4, ...), every warp runs all MT row tiles; blockIdx.y is the K split.  The
//   adapter's bytes are read once per row tile.  No atomics: split p writes its own partial y[p].
// * Expand: the CTA sums the partials of its rows in split order (a fixed order, so results are bitwise reproducible)
//   into shared memory as bf16, then the warps split 128 output columns (4 n8 tiles each) with R as the contraction.
//   Each output element belongs to one lane, which reads, adds and writes it.
#include "kernels.h"

namespace ab {

constexpr int kLoraThreads = 128;
constexpr int kLoraWarps = kLoraThreads / 32;
constexpr int kShrinkTiles = kLoraMaxRank / 8 / kLoraWarps;  // n8 tiles of R per warp in shrink
constexpr int kExpandTiles = 4;                              // n8 tiles of N per warp in expand
constexpr int kExpandCols = kLoraWarps * kExpandTiles * 8;   // output columns per expand CTA

__device__ __forceinline__ void mma16816(float* d, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Two MMAs over one 32-wide k step: xa[h] holds 8 k values of row g + 8h, wb 8 k values of column g.
__device__ __forceinline__ void mma_k32(float* d, const uint4* xa, const uint4& wb) {
  mma16816(d, xa[0].x, xa[1].x, xa[0].y, xa[1].y, wb.x, wb.y);
  mma16816(d, xa[0].z, xa[1].z, xa[0].w, xa[1].w, wb.z, wb.w);
}

// The segment and rows [r0, r1) of row tile `tile`; false past the last tile.
__device__ __forceinline__ bool find_tile(const LoraArgs& a, int BM, int tile, int& seg, int& r0, int& r1) {
  for (int s = 0; s < a.S; ++s) {
    const int b = a.seg_start[s], e = a.seg_start[s + 1];
    const int n = e > b ? (e - b + BM - 1) / BM : 0;
    if (tile < n) {
      seg = s;
      r0 = b + tile * BM;
      r1 = min(e, r0 + BM);
      return true;
    }
    tile -= n;
  }
  return false;
}

template <int MT>
__global__ void __launch_bounds__(kLoraThreads) lora_shrink_sm90_kernel(const LoraArgs a) {
  int seg, r0, r1;
  if (!find_tile(a, 16 * MT, blockIdx.x, seg, r0, r1)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const __nv_bfloat16* A = a.w + (long long)a.seg_slot[seg] * a.R * a.K;
  const int kper = (a.K + 32 * a.splits - 1) / (32 * a.splits) * 32;
  const int k0 = blockIdx.y * kper, k1 = min(a.K, k0 + kper);
  const int ntiles = a.R / 8;

  const __nv_bfloat16* xr[MT][2];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = r0 + m * 16 + h * 8 + g;
      xr[m][h] = i < r1 ? a.x + (long long)a.rows[i] * a.ldx : nullptr;
    }
  float acc[MT][kShrinkTiles][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int j = 0; j < kShrinkTiles; ++j) acc[m][j][0] = acc[m][j][1] = acc[m][j][2] = acc[m][j][3] = 0.f;

  const uint4 zero = make_uint4(0, 0, 0, 0);
#pragma unroll 2
  for (int kb = k0; kb < k1; kb += 32) {
    const int k = kb + 8 * q;
    const bool kin = k < k1;                 // K is a multiple of 8: a lane's 8 values are all in or all out
    uint4 xa[MT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        xa[m][h] = kin && xr[m][h] ? __ldg(reinterpret_cast<const uint4*>(xr[m][h] + k)) : zero;
#pragma unroll
    for (int j = 0; j < kShrinkTiles; ++j) {
      const int t = warp + j * kLoraWarps;
      if (t >= ntiles) break;                // warp-uniform
      const uint4 wb = kin ? __ldg(reinterpret_cast<const uint4*>(A + (long long)(t * 8 + g) * a.K + k)) : zero;
#pragma unroll
      for (int m = 0; m < MT; ++m) mma_k32(acc[m][j], xa[m], wb);
    }
  }

  float* y = a.y + (long long)blockIdx.y * a.Tl * a.R;
#pragma unroll
  for (int j = 0; j < kShrinkTiles; ++j) {
    const int t = warp + j * kLoraWarps;
    if (t >= ntiles) break;
    const int n = t * 8 + 2 * q;
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = r0 + m * 16 + h * 8 + g;
        if (i < r1) *reinterpret_cast<float2*>(y + (long long)i * a.R + n) = make_float2(acc[m][j][2 * h], acc[m][j][2 * h + 1]);
      }
  }
}

// Shared row stride of the staged y tile: at least R rounded up to 32, and 32 mod 64 elements so the 8 lanes of a
// 16-byte load phase (rows g, g + 1, four k offsets) hit distinct banks.
__host__ __device__ constexpr int expand_ld(int R) { return (R + 31) / 64 * 64 + 32; }

template <int MT>
__global__ void __launch_bounds__(kLoraThreads) lora_expand_sm90_kernel(const LoraArgs a) {
  constexpr int BM = 16 * MT;
  __shared__ __align__(16) __nv_bfloat16 ys[BM * expand_ld(kLoraMaxRank)];
  int seg, r0, r1;
  if (!find_tile(a, BM, blockIdx.y, seg, r0, r1)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int slot = a.seg_slot[seg];
  const int Rp = (a.R + 31) / 32 * 32, ld = expand_ld(a.R);

  // y rows of the tile, split partials summed in order p = 0, 1, ..; zero past the segment and past R
  for (int e = threadIdx.x; e < BM * (Rp / 4); e += kLoraThreads) {
    const int r = e / (Rp / 4), c = (e % (Rp / 4)) * 4;
    const int i = r0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < r1 && c < a.R) {
      const float* p = a.y + (long long)i * a.R + c;
      for (int s = 0; s < a.splits; ++s, p += (long long)a.Tl * a.R) {
        const float4 t = *reinterpret_cast<const float4*>(p);
        v.x += t.x;
        v.y += t.y;
        v.z += t.z;
        v.w += t.w;
      }
    }
    __nv_bfloat162* d = reinterpret_cast<__nv_bfloat162*>(ys + r * ld + c);
    d[0] = __floats2bfloat162_rn(v.x, v.y);
    d[1] = __floats2bfloat162_rn(v.z, v.w);
  }
  __syncthreads();

  const __nv_bfloat16* B = a.w + (long long)slot * a.N * a.R;
  const int n0 = blockIdx.x * kExpandCols + warp * kExpandTiles * 8;
  const __nv_bfloat16* br[kExpandTiles];
#pragma unroll
  for (int j = 0; j < kExpandTiles; ++j) {
    const int n = n0 + j * 8 + g;
    br[j] = n < a.N ? B + (long long)n * a.R : nullptr;
  }
  float acc[MT][kExpandTiles][4];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int j = 0; j < kExpandTiles; ++j) acc[m][j][0] = acc[m][j][1] = acc[m][j][2] = acc[m][j][3] = 0.f;

  const uint4 zero = make_uint4(0, 0, 0, 0);
  for (int kb = 0; kb < Rp; kb += 32) {
    const int k = kb + 8 * q;
    uint4 wb[kExpandTiles];
#pragma unroll
    for (int j = 0; j < kExpandTiles; ++j)
      wb[j] = k < a.R && br[j] ? __ldg(reinterpret_cast<const uint4*>(br[j] + k)) : zero;
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      uint4 ya[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) ya[h] = *reinterpret_cast<const uint4*>(ys + (m * 16 + h * 8 + g) * ld + k);
#pragma unroll
      for (int j = 0; j < kExpandTiles; ++j) mma_k32(acc[m][j], ya, wb[j]);
    }
  }

  const float s = a.scale[slot];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = r0 + m * 16 + h * 8 + g;
      if (i >= r1) continue;
      __nv_bfloat16* o = a.out + (long long)a.rows[i] * a.ldo;
#pragma unroll
      for (int j = 0; j < kExpandTiles; ++j) {
        const int n = n0 + j * 8 + 2 * q;
        if (n >= a.N) continue;
        __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(o + n);
        const float2 cur = __bfloat1622float2(*p);
        *p = __floats2bfloat162_rn(cur.x + s * acc[m][j][2 * h], cur.y + s * acc[m][j][2 * h + 1]);
      }
    }
}

// MT = 4 when the segments average 48 rows or more (prefill), else 1 (decode: a few rows per adapter).
static bool wide_tiles(const LoraArgs& a) { return a.Tl >= 48 * a.S; }

static long long row_tiles(const LoraArgs& a, int BM) { return (a.Tl + BM - 1) / BM + a.S; }

}  // namespace ab

extern "C" int ab_lora_splits(const ab::LoraArgs* a) {
  using namespace ab;
  if (a->Tl <= 0 || a->S <= 0 || a->K <= 0) return 1;
  const long long tiles = row_tiles(*a, wide_tiles(*a) ? 64 : 16);
  // about two CTAs per SM, each split at least 512 columns of K
  const long long splits = (2LL * num_sms() + tiles - 1) / tiles, cap = a->K / 512 > 1 ? a->K / 512 : 1;
  return (int)(splits > cap ? cap : splits);
}

extern "C" int ab_lora_shrink(const ab::LoraArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->R <= 0 || a->R > kLoraMaxRank || a->R % 8 || a->K % 8 || a->splits < 1) return 1;
  if (a->Tl == 0 || a->S == 0) return 0;
  const bool wide = wide_tiles(*a);
  const long long tiles = row_tiles(*a, wide ? 64 : 16);
  if (tiles > 0x7fffffffLL || a->splits > 65535) return 2;
  const dim3 grid((unsigned)tiles, a->splits);
  if (wide)
    lora_shrink_sm90_kernel<4><<<grid, kLoraThreads, 0, st>>>(*a);
  else
    lora_shrink_sm90_kernel<1><<<grid, kLoraThreads, 0, st>>>(*a);
  return cudaGetLastError() == cudaSuccess ? 0 : 30;
}

extern "C" int ab_lora_expand(const ab::LoraArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->R <= 0 || a->R > kLoraMaxRank || a->R % 8 || a->N % 8 || a->splits < 1) return 1;
  if (a->Tl == 0 || a->S == 0 || a->N == 0) return 0;
  const bool wide = wide_tiles(*a);
  const long long tiles = row_tiles(*a, wide ? 64 : 16);
  if (tiles > 65535) return 2;
  const dim3 grid((unsigned)((a->N + kExpandCols - 1) / kExpandCols), (unsigned)tiles);
  if (wide)
    lora_expand_sm90_kernel<4><<<grid, kLoraThreads, 0, st>>>(*a);
  else
    lora_expand_sm90_kernel<1><<<grid, kLoraThreads, 0, st>>>(*a);
  return cudaGetLastError() == cudaSuccess ? 0 : 30;
}
