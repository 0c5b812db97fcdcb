// Fused softmax-attention forward and backward for sm_90a (K2 of SURVEY.md §2.5).
//
// Reference behaviour: softmax(Q K^T / sqrt(d) [+ causal mask]) V with the [B,h,S,S] score tensor
// materialised by two cuBLAS batched GEMMs + an XLA softmax fusion (alpa/model/bert_model.py:203-217).
//
// All products run on wgmma with fp32 accumulators in warpgroup registers; tiles arrive by TMA (128-byte swizzle,
// [rows][64 head-dim elements] atoms) into a two-stage shared-memory ring guarded by mbarriers.  Every product is one
// of two forms:
//   SS  X[64 rows] . Y^T, contraction over the head dim: both operands K-major descriptors   (S = Q K^T, dP = dO V^T)
//   RS  F[64 rows] . Z,   contraction over tile rows: F in registers (the mma.sync A-fragment layout, converted
//       straight from the previous accumulator), Z an MN-major descriptor                      (O += P V, dQ += dS K, ...)
//
// Forward: one CTA per (batch, head, 64 x WG query rows), one warpgroup per 64 rows, K/V tiles of 64 keys; online
//   softmax in exp2 form with P kept in registers.
// Backward: two kernels without atomics, so the gradients are the same from run to run.  dK / dV: one warpgroup per
//   (batch, head, 64-key tile) holding dK / dV in registers while Q / dO tiles stream through the ring
//   (S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q).  dQ: one warpgroup per 64 query rows with the forward's
//   structure (S = Q K^T, dP = dO V^T, dQ += dS K).
//
// Grouped-query attention: query head hq = kv * group + g reads K/V head kv.  Forward and dQ CTAs take the K/V tiles of
//   their query head's K/V head, and the G CTAs of one query tile of a group are adjacent in the grid, so they read the
//   same K/V tiles at about the same time (from L2).  dK / dV: one warpgroup per (batch, K/V head, 64-key tile) streams
//   the (Q, dO) tiles of every query head of the group through the ring and accumulates over all of them in registers.
//   When those CTAs are too few to fill the GPU, the group is split into parts (ab_attention_bwd_splits) that write
//   fp32 partials; attn_bwd_dkdv_reduce_kernel sums them in a fixed order.
//
// Masking (both directions): key j is visible to query i iff j < Skv and, when causal, j <= i + (Skv - Sq); Skv is the
// device-side kv_len when one is given.  Head dims up to 128 in multiples of 8 run as 64 or 128 (TMA zero-fills).
#include "kernels.h"
#include "attention_sm90.cuh"
#include "tma_host.h"

namespace ab {

// Loads tile rows [row0, row0 + rows) of a [B, S, heads, D] tensor map into DP / 64 atoms of rows x 128 B.
template <int DP>
__device__ __forceinline__ void tma_tile(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int row0, int rows, int h,
                                         int b) {
#pragma unroll
  for (int at = 0; at < DP / 64; ++at) tma_load_4d(dst + at * rows * 128, m, bar, at * 64, row0, h, b);
}
// The same from a [B, S, kv_heads, group, D] (query) tensor map.
template <int DP>
__device__ __forceinline__ void tma_tile_q(uint8_t* dst, const CUtensorMap* m, uint64_t* bar, int row0, int rows,
                                           int g, int kv, int b) {
#pragma unroll
  for (int at = 0; at < DP / 64; ++at) tma_load_5d(dst + at * rows * 128, m, bar, at * 64, row0, g, kv, b);
}

// ------------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------------
template <int DP, int WG>
struct AttnFwdSmem {
  static constexpr int kQ = (DP / 64) * (64 * WG) * 128;
  static constexpr int kKV = (DP / 64) * kAtomRows64;  // one K or V tile
  static constexpr int kTotal = kQ + 4 * kKV + 64 + 1024;
};

template <int DP, int WG>
__global__ void __launch_bounds__(WG * 128, 1)
attn_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                     const __grid_constant__ CUtensorMap tv, const AttnArgs a, float scale_log2) {
  using L = AttnFwdSmem<DP, WG>;
  constexpr int kBQ = 64 * WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + L::kQ;  // stage s: K at sKV + 2 s kKV, V right after
  uint64_t* bar = reinterpret_cast<uint64_t*>(sKV + 4 * L::kKV);  // [0] Q, [1 + s] K/V stage s

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int wi = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int G = a.group;
  const int qt = blockIdx.x / G, gq = blockIdx.x - qt * G;  // x = query tile * G + head within the group
  const int b = blockIdx.y / a.kv_heads, kvh = blockIdx.y - b * a.kv_heads;
  const int hq = kvh * G + gq;
  const int q0 = qt * kBQ;
  const int Skv = a.kv_len != nullptr ? min(a.Skv, *a.kv_len) : a.Skv;
  const int shift = Skv - a.Sq;  // causal: key j visible to query i iff j <= i + shift
  int kv_end = Skv;
  if (a.causal) kv_end = min(Skv, q0 + kBQ + shift);
  const int n_tiles = kv_end > 0 ? (kv_end + kTile - 1) / kTile : 0;

  auto issue_kv = [&](int j) {
    const int s = j & 1;
    mbar_expect_tx(&bar[1 + s], 2 * L::kKV);
    tma_tile<DP>(sKV + 2 * s * L::kKV, &tk, &bar[1 + s], j * kTile, kTile, kvh, b);
    tma_tile<DP>(sKV + (2 * s + 1) * L::kKV, &tv, &bar[1 + s], j * kTile, kTile, kvh, b);
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    mbar_fence_init();
    mbar_expect_tx(&bar[0], L::kQ);
    tma_tile_q<DP>(sQ, &tq, &bar[0], q0, kBQ, gq, kvh, b);
    for (int j = 0; j < 2 && j < n_tiles; ++j) issue_kv(j);
  }
  __syncthreads();

  float o[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  const int row0 = q0 + wg * 64 + wi * 16;  // first query row of this warp
  const int qrow[2] = {row0 + g, row0 + g + 8};
  const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;
  mbar_wait(&bar[0], 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j & 1;
    mbar_wait(&bar[1 + s], (j >> 1) & 1);
    const uint32_t sk = smem_u32(sKV + 2 * s * L::kKV), sv = sk + L::kKV;
    const int kv0 = j * kTile;

    float sc[8][4];  // S = Q K^T: the 16 x 64 block of this warp
    wgmma_fence();
    mma_ss_64<DP>(&sc[0][0], q_addr, kBQ * 128, sk, kAtomRows64);
    mma_sync_all();

    // scale to exp2 and mask: key j is visible to query i iff j < Skv and, when causal, j <= i + shift
    const bool need_mask = kv0 + kTile > Skv || (a.causal && kv0 + kTile - 1 > row0 + shift);
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[n][e] * scale_log2;
        if (need_mask) {
          const int key = kv0 + n * 8 + 2 * t + (e & 1);
          if (key >= Skv || (a.causal && key > qrow[e >> 1] + shift)) v = -INFINITY;
        }
        sc[n][e] = v;
      }
    }
    fwd_softmax_pv<DP>(sc, o, m_r, l_r, sv);
    __syncthreads();  // every warpgroup is done with stage s: refill it with tile j + 2
    if (threadIdx.x == 0 && j + 2 < n_tiles) issue_kv(j + 2);
  }

  // epilogue: O / l, lse = (m + log2 l) ln 2
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_r[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qi = qrow[r];
    const float inv = l > 0.f ? 1.f / l : 0.f;
    if (qi < a.Sq) {
      __nv_bfloat16* og = a.o + (long long)b * a.o_stride_b + (long long)qi * a.o_stride_s + (long long)hq * a.o_stride_h;
#pragma unroll
      for (int dn = 0; dn < DP / 8; ++dn) {
        const int d = dn * 8 + 2 * t;
        if (d < a.D)
          *reinterpret_cast<uint32_t*>(og + d) = pack_bf16x2(o[dn][2 * r] * inv, o[dn][2 * r + 1] * inv);
      }
      if (t == 0)
        a.lse[((long long)b * a.kv_heads * G + hq) * a.Sq + qi] = l > 0.f ? (m_r[r] + __log2f(l)) * 0.69314718055994531f : -INFINITY;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------
template <int DP>
struct AttnBwdSmem {
  static constexpr int kT = (DP / 64) * kAtomRows64;  // one [64 rows][DP] tile
  static constexpr int kTotal = 6 * kT + 64 + 1024;   // two resident tiles + a two-stage ring of two tiles
};

// dK / dV of 64 keys: K, V resident, (Q, dO) tiles of 64 queries through the ring, for query heads [g0, g1) of the
// group (part blockIdx.z of a.splits).  One part writes bf16; several write fp32 partials for the reduce kernel.
template <int DP>
__global__ void __launch_bounds__(128, 1)
attn_bwd_dkdv_sm90_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                          const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo,
                          const AttnBwdArgs a, float scale_log2) {
  using L = AttnBwdSmem<DP>;
  const AttnArgs& f = a.f;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sK = smem;
  uint8_t* sV = smem + L::kT;
  uint8_t* sRing = smem + 2 * L::kT;  // stage s: Q at sRing + 2 s kT, dO right after
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 6 * L::kT);  // [0] K/V, [1 + s] ring stage s

  const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int G = f.group;
  const int b = blockIdx.y / f.kv_heads, kvh = blockIdx.y - b * f.kv_heads;
  const int g0 = blockIdx.z * G / a.splits, g1 = (blockIdx.z + 1) * G / a.splits;
  const int kv0 = blockIdx.x * kTile;
  const int Sq = f.Sq, Skv = f.Skv, shift = Skv - Sq;
  const int qt0 = (f.causal ? max(0, kv0 - shift) : 0) / kTile;
  const int q_tiles = max(0, (Sq + kTile - 1) / kTile - qt0);  // per query head
  const int n_tiles = (g1 - g0) * q_tiles;                       // step i: head g0 + i / q_tiles, tile i % q_tiles

  auto issue_q = [&](int i) {
    const int s = i & 1;
    const int gh = g0 + i / q_tiles, q0 = (qt0 + i % q_tiles) * kTile;
    mbar_expect_tx(&bar[1 + s], 2 * L::kT);
    tma_tile_q<DP>(sRing + 2 * s * L::kT, &tq, &bar[1 + s], q0, kTile, gh, kvh, b);
    tma_tile<DP>(sRing + (2 * s + 1) * L::kT, &tdo, &bar[1 + s], q0, kTile, kvh * G + gh, b);
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    mbar_fence_init();
    mbar_expect_tx(&bar[0], 2 * L::kT);
    tma_tile<DP>(sK, &tk, &bar[0], kv0, kTile, kvh, b);
    tma_tile<DP>(sV, &tv, &bar[0], kv0, kTile, kvh, b);
    for (int i = 0; i < 2 && i < n_tiles; ++i) issue_q(i);
  }
  __syncthreads();

  float dk[DP / 8][4], dv[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[i][e] = dv[i][e] = 0.f;
  const int key_row[2] = {kv0 + wi * 16 + g, kv0 + wi * 16 + g + 8};
  const uint32_t k_addr = smem_u32(sK), v_addr = smem_u32(sV);
  mbar_wait(&bar[0], 0);

  for (int i = 0; i < n_tiles; ++i) {
    const int s = i & 1;
    const int gh = g0 + i / q_tiles;
    const int q0 = (qt0 + i - (gh - g0) * q_tiles) * kTile;
    const long long stat_row = ((long long)b * f.kv_heads * G + kvh * G + gh) * Sq;
    const float* lse = f.lse + stat_row;
    const float* delta = a.delta + stat_row;
    // per-query statistics of the 16 score columns this thread holds
    float lse2[8][2], dl[8][2];
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int qi = q0 + n * 8 + 2 * t + c;
        lse2[n][c] = qi < Sq ? lse[qi] * 1.4426950408889634f : INFINITY;  // P = 0 for padding queries
        dl[n][c] = qi < Sq ? delta[qi] : 0.f;
      }
    mbar_wait(&bar[1 + s], (i >> 1) & 1);
    const uint32_t sq = smem_u32(sRing + 2 * s * L::kT), sdo = sq + L::kT;

    float st[8][4], dpt[8][4];  // S^T = K Q^T and dP^T = V dO^T: 16 keys x 64 queries per warp
    wgmma_fence();
    mma_ss_64<DP>(&st[0][0], k_addr, kAtomRows64, sq, kAtomRows64);
    mma_ss_64<DP>(&dpt[0][0], v_addr, kAtomRows64, sdo, kAtomRows64);
    mma_sync_all();

    uint32_t pt[4][4], dst[4][4];  // P^T and dS^T = P^T (dP^T - delta) (scale folded into dK)
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      float p[4], ds[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = q0 + n * 8 + 2 * t + (e & 1);
        const int key = key_row[e >> 1];
        const bool vis = key < Skv && (!f.causal || key <= qi + shift);
        p[e] = vis ? ex2_approx(st[n][e] * scale_log2 - lse2[n][e & 1]) : 0.f;
        ds[e] = p[e] * (dpt[n][e] - dl[n][e & 1]);
      }
      pt[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p[0], p[1]);
      pt[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(p[2], p[3]);
      dst[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(ds[0], ds[1]);
      dst[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(ds[2], ds[3]);
    }
    wgmma_fence();
    mma_rs<DP>(&dv[0][0], pt, sdo, kAtomRows64);   // dV += P^T dO
    mma_rs<DP>(&dk[0][0], dst, sq, kAtomRows64);   // dK += dS^T Q
    mma_sync_all();
    __syncthreads();
    if (threadIdx.x == 0 && i + 2 < n_tiles) issue_q(i + 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_row[r];
    if (key >= Skv) continue;
    if (a.splits > 1) {
      const long long dv_off = (long long)a.splits * f.B * f.kv_heads * Skv * f.D;  // dK partials, then dV partials
      float* wk = a.ws + ((((long long)blockIdx.z * f.B + b) * f.kv_heads + kvh) * Skv + key) * f.D;
#pragma unroll
      for (int dn = 0; dn < DP / 8; ++dn) {
        const int d = dn * 8 + 2 * t;
        if (d < f.D) {
          *reinterpret_cast<float2*>(wk + d) = make_float2(dk[dn][2 * r], dk[dn][2 * r + 1]);
          *reinterpret_cast<float2*>(wk + dv_off + d) = make_float2(dv[dn][2 * r], dv[dn][2 * r + 1]);
        }
      }
      continue;
    }
    __nv_bfloat16* dkg = a.dk + (long long)b * a.dk_stride_b + (long long)key * a.dk_stride_s + (long long)kvh * a.dk_stride_h;
    __nv_bfloat16* dvg = a.dv + (long long)b * a.dv_stride_b + (long long)key * a.dv_stride_s + (long long)kvh * a.dv_stride_h;
#pragma unroll
    for (int dn = 0; dn < DP / 8; ++dn) {
      const int d = dn * 8 + 2 * t;
      if (d < f.D) {
        *reinterpret_cast<uint32_t*>(dkg + d) = pack_bf16x2(dk[dn][2 * r] * f.scale, dk[dn][2 * r + 1] * f.scale);
        *reinterpret_cast<uint32_t*>(dvg + d) = pack_bf16x2(dv[dn][2 * r], dv[dn][2 * r + 1]);
      }
    }
  }
}

// dK / dV of a split group: the sum of the splits' fp32 partials in part order (fixed, so the result is the same from
// run to run), dK scaled, rounded to bf16 once.  One thread per two adjacent head-dim elements.
__global__ void attn_bwd_dkdv_reduce_kernel(const AttnBwdArgs a) {
  const AttnArgs& f = a.f;
  const int half_d = f.D / 2;
  const long long n = (long long)f.B * f.kv_heads * f.Skv * half_d;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int d = (int)(i % half_d) * 2;
  const long long row = i / half_d;  // (b, kv, key)
  const int key = (int)(row % f.Skv);
  const int kvh = (int)((row / f.Skv) % f.kv_heads);
  const int b = (int)(row / ((long long)f.Skv * f.kv_heads));
  const long long part = n * 2, dv_off = (long long)a.splits * part;
  float2 sk = make_float2(0.f, 0.f), sv = make_float2(0.f, 0.f);
  for (int p = 0; p < a.splits; ++p) {
    const float2 x = *reinterpret_cast<const float2*>(a.ws + p * part + row * f.D + d);
    const float2 y = *reinterpret_cast<const float2*>(a.ws + dv_off + p * part + row * f.D + d);
    sk.x += x.x; sk.y += x.y;
    sv.x += y.x; sv.y += y.y;
  }
  __nv_bfloat16* dkg = a.dk + (long long)b * a.dk_stride_b + (long long)key * a.dk_stride_s + (long long)kvh * a.dk_stride_h;
  __nv_bfloat16* dvg = a.dv + (long long)b * a.dv_stride_b + (long long)key * a.dv_stride_s + (long long)kvh * a.dv_stride_h;
  *reinterpret_cast<uint32_t*>(dkg + d) = pack_bf16x2(sk.x * f.scale, sk.y * f.scale);
  *reinterpret_cast<uint32_t*>(dvg + d) = pack_bf16x2(sv.x, sv.y);
}

// dQ of 64 queries: Q, dO resident, (K, V) tiles through the ring.
template <int DP>
__global__ void __launch_bounds__(128, 1)
attn_bwd_dq_sm90_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                        const __grid_constant__ CUtensorMap tv, const __grid_constant__ CUtensorMap tdo,
                        const AttnBwdArgs a, float scale_log2) {
  using L = AttnBwdSmem<DP>;
  const AttnArgs& f = a.f;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sDO = smem + L::kT;
  uint8_t* sRing = smem + 2 * L::kT;  // stage s: K at sRing + 2 s kT, V right after
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 6 * L::kT);

  const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int G = f.group;
  const int qt = blockIdx.x / G, gq = blockIdx.x - qt * G;  // x = query tile * G + head within the group
  const int b = blockIdx.y / f.kv_heads, kvh = blockIdx.y - b * f.kv_heads;
  const int hq = kvh * G + gq;
  const int q0 = qt * kTile;
  const int Skv = f.Skv, shift = Skv - f.Sq;
  int kv_end = Skv;
  if (f.causal) kv_end = min(Skv, q0 + kTile + shift);
  const int n_tiles = kv_end > 0 ? (kv_end + kTile - 1) / kTile : 0;

  auto issue_kv = [&](int j) {
    const int s = j & 1;
    mbar_expect_tx(&bar[1 + s], 2 * L::kT);
    tma_tile<DP>(sRing + 2 * s * L::kT, &tk, &bar[1 + s], j * kTile, kTile, kvh, b);
    tma_tile<DP>(sRing + (2 * s + 1) * L::kT, &tv, &bar[1 + s], j * kTile, kTile, kvh, b);
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    mbar_fence_init();
    mbar_expect_tx(&bar[0], 2 * L::kT);
    tma_tile_q<DP>(sQ, &tq, &bar[0], q0, kTile, gq, kvh, b);
    tma_tile<DP>(sDO, &tdo, &bar[0], q0, kTile, hq, b);
    for (int j = 0; j < 2 && j < n_tiles; ++j) issue_kv(j);
  }
  __syncthreads();

  const int row0 = q0 + wi * 16;
  const int qrow[2] = {row0 + g, row0 + g + 8};
  float lse2[2], dlt[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const bool ok = qrow[r] < f.Sq;
    const long long idx = ((long long)b * f.kv_heads * G + hq) * f.Sq + qrow[r];
    lse2[r] = ok ? f.lse[idx] * 1.4426950408889634f : INFINITY;
    dlt[r] = ok ? a.delta[idx] : 0.f;
  }
  float dq[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  const uint32_t q_addr = smem_u32(sQ), do_addr = smem_u32(sDO);
  mbar_wait(&bar[0], 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j & 1;
    mbar_wait(&bar[1 + s], (j >> 1) & 1);
    const uint32_t sk = smem_u32(sRing + 2 * s * L::kT), sv = sk + L::kT;
    const int kv0 = j * kTile;
    float sc[8][4], dp[8][4];  // S = Q K^T, dP = dO V^T
    wgmma_fence();
    mma_ss_64<DP>(&sc[0][0], q_addr, kAtomRows64, sk, kAtomRows64);
    mma_ss_64<DP>(&dp[0][0], do_addr, kAtomRows64, sv, kAtomRows64);
    mma_sync_all();
    uint32_t dsf[4][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      float ds[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kv0 + n * 8 + 2 * t + (e & 1);
        const bool vis = key < Skv && (!f.causal || key <= qrow[e >> 1] + shift);
        const float p = vis ? ex2_approx(sc[n][e] * scale_log2 - lse2[e >> 1]) : 0.f;
        ds[e] = p * (dp[n][e] - dlt[e >> 1]);
      }
      dsf[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(ds[0], ds[1]);
      dsf[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(ds[2], ds[3]);
    }
    wgmma_fence();
    mma_rs<DP>(&dq[0][0], dsf, sk, kAtomRows64);  // dQ += dS K
    mma_sync_all();
    __syncthreads();
    if (threadIdx.x == 0 && j + 2 < n_tiles) issue_kv(j + 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = qrow[r];
    if (qi >= f.Sq) continue;
    __nv_bfloat16* dqg = a.dq + (long long)b * a.dq_stride_b + (long long)qi * a.dq_stride_s + (long long)kvh * a.dq_stride_h +
                         (long long)gq * a.dq_stride_g;
#pragma unroll
    for (int dn = 0; dn < DP / 8; ++dn) {
      const int d = dn * 8 + 2 * t;
      if (d < f.D)
        *reinterpret_cast<uint32_t*>(dqg + d) = pack_bf16x2(dq[dn][2 * r] * f.scale, dq[dn][2 * r + 1] * f.scale);
    }
  }
}

// delta[b,h,q] = sum_d dO[b,q,h,d] * O[b,q,h,d]; GW lanes (one 16-byte load each) per (b,q,h) row.
template <int GW>
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                                  float* __restrict__ delta, int B, int H, int Sq, int D,
                                  long long sb, long long ss, long long sh) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long w = gid / GW;
  const int part = (int)(gid % GW);
  const bool valid = w < (long long)B * Sq * H;
  float acc = 0.f;
  int h = 0, q = 0, b = 0;
  if (valid) {
    h = (int)(w % H);
    q = (int)((w / H) % Sq);
    b = (int)(w / ((long long)H * Sq));
    if (part * 8 < D) {
      const size_t base = (size_t)b * sb + (size_t)q * ss + (size_t)h * sh + part * 8;
      const int4 x = ld_nc_v4(d_o + base);
      const int4 c = ld_nc_v4(o + base);
      const uint32_t* xu = reinterpret_cast<const uint32_t*>(&x);
      const uint32_t* cu = reinterpret_cast<const uint32_t*>(&c);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fa = unpack_bf16x2(xu[j]), fc = unpack_bf16x2(cu[j]);
        acc += fa.x * fc.x + fa.y * fc.y;
      }
    }
  }
#pragma unroll
  for (int o2 = GW / 2; o2 > 0; o2 >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o2);
  if (valid && part == 0) delta[((size_t)b * H + h) * Sq + q] = acc;
}

// tensor map of a [B, S, heads, D] view (D contiguous), box of 64 head-dim elements x `rows`
static int make_qkv_tmap(CUtensorMap* m, const __nv_bfloat16* p, int D, int S, int H, int B, long long ss,
                         long long sh, long long sb, int rows) {
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)S, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)ss, (uint64_t)sh, (uint64_t)sb};
  return make_tmap_bf16_4d(m, p, dims, strides, 64, rows);
}

// tensor map of the query view [B, S, kv_heads, group, D]; a group of one takes the K/V-head stride for its (only ever
// zero) group coordinate, since a size-1 dim's stride can be anything
static int make_q_tmap(CUtensorMap* m, const AttnArgs& a, int rows) {
  const uint64_t dims[5] = {(uint64_t)a.D, (uint64_t)a.Sq, (uint64_t)a.group, (uint64_t)a.kv_heads, (uint64_t)a.B};
  const uint64_t strides[4] = {(uint64_t)a.q_stride_s, (uint64_t)(a.group > 1 ? a.q_stride_g : a.q_stride_h),
                               (uint64_t)a.q_stride_h, (uint64_t)a.q_stride_b};
  return make_tmap_bf16_5d(m, a.q, dims, strides, 64, rows);
}

template <typename Kern>
static bool set_smem(Kern k, int bytes) {
  return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess;
}

template <int DP, int WG>
static int attn_fwd_launch(const AttnArgs& a, cudaStream_t st) {
  CUtensorMap tq, tk, tv;
  if (make_q_tmap(&tq, a, 64 * WG)) return 10;
  if (make_qkv_tmap(&tk, a.k, a.D, a.Skv, a.kv_heads, a.B, a.k_stride_s, a.k_stride_h, a.k_stride_b, kTile)) return 11;
  if (make_qkv_tmap(&tv, a.v, a.D, a.Skv, a.kv_heads, a.B, a.v_stride_s, a.v_stride_h, a.v_stride_b, kTile)) return 12;
  auto kern = attn_fwd_sm90_kernel<DP, WG>;
  constexpr int smem = AttnFwdSmem<DP, WG>::kTotal;
  static bool attr_set = false;
  if (!attr_set) {
    if (!set_smem(kern, smem)) return 20;
    attr_set = true;
  }
  dim3 grid((a.Sq + 64 * WG - 1) / (64 * WG) * a.group, a.B * a.kv_heads);
  kern<<<grid, WG * 128, smem, st>>>(tq, tk, tv, a, a.scale * 1.4426950408889634f);
  return cudaGetLastError() == cudaSuccess ? 0 : 30;
}

// Parts the dK / dV kernel splits each group of query heads into.  Its grid has B * kv_heads * ceil(Skv / 64) CTAs of
// one warpgroup, and each holds about 97 KB of shared memory at head dim 128 (half at 64), so two or more share an SM.
// When the grid is short of two CTAs per SM (grouped heads at tensor-parallel shapes: one K/V head per GPU), the group
// is split into P parts, P the smallest divisor of the group size that gives at least 2 x SMs CTAs (else the whole
// group, one head per CTA).  Equal parts keep the CTAs' work equal.  P > 1 costs one fp32 partial of dK and dV per part
// and a reduce kernel; multi-head attention (group 1) never splits.
static int bwd_splits(const AttnArgs& f) {
  const long long ctas = (long long)f.B * f.kv_heads * ((f.Skv + kTile - 1) / kTile);
  const long long want = 2LL * num_sms();
  for (int p = 1; p < f.group; ++p)
    if (f.group % p == 0 && ctas * p >= want) return p;
  return f.group;
}

template <int DP>
static int attn_bwd_launch(const AttnBwdArgs& a, cudaStream_t st) {
  const AttnArgs& f = a.f;
  const int Hq = f.kv_heads * f.group;
  CUtensorMap tq, tk, tv, tdo;
  if (make_q_tmap(&tq, f, kTile)) return 10;
  if (make_qkv_tmap(&tk, f.k, f.D, f.Skv, f.kv_heads, f.B, f.k_stride_s, f.k_stride_h, f.k_stride_b, kTile)) return 11;
  if (make_qkv_tmap(&tv, f.v, f.D, f.Skv, f.kv_heads, f.B, f.v_stride_s, f.v_stride_h, f.v_stride_b, kTile)) return 12;
  if (make_qkv_tmap(&tdo, a.d_o, f.D, f.Sq, Hq, f.B, f.o_stride_s, f.o_stride_h, f.o_stride_b, kTile)) return 13;
  if (a.splits < 1 || a.splits > f.group || (a.splits > 1 && a.ws == nullptr)) return 14;
  auto kern = attn_bwd_dkdv_sm90_kernel<DP>;
  auto kern_dq = attn_bwd_dq_sm90_kernel<DP>;
  constexpr int smem = AttnBwdSmem<DP>::kTotal;
  static bool attr_set = false;
  if (!attr_set) {
    if (!set_smem(kern, smem) || !set_smem(kern_dq, smem)) return 20;
    attr_set = true;
  }
  const int rows = f.B * f.Sq * Hq;
  if (f.D <= 64)
    attn_delta_kernel<8><<<(int)(((long long)rows * 8 + 255) / 256), 256, 0, st>>>(
        a.d_o, f.o, a.delta, f.B, Hq, f.Sq, f.D, f.o_stride_b, f.o_stride_s, f.o_stride_h);
  else
    attn_delta_kernel<16><<<(int)(((long long)rows * 16 + 255) / 256), 256, 0, st>>>(
        a.d_o, f.o, a.delta, f.B, Hq, f.Sq, f.D, f.o_stride_b, f.o_stride_s, f.o_stride_h);
  const float sl2 = f.scale * 1.4426950408889634f;
  kern<<<dim3((f.Skv + kTile - 1) / kTile, f.B * f.kv_heads, a.splits), 128, smem, st>>>(tq, tk, tv, tdo, a, sl2);
  if (cudaGetLastError() != cudaSuccess) return 30;
  if (a.splits > 1) {
    const long long n = (long long)f.B * f.kv_heads * f.Skv * (f.D / 2);
    attn_bwd_dkdv_reduce_kernel<<<(int)((n + 255) / 256), 256, 0, st>>>(a);
    if (cudaGetLastError() != cudaSuccess) return 32;
  }
  kern_dq<<<dim3((f.Sq + kTile - 1) / kTile * f.group, f.B * f.kv_heads), 128, smem, st>>>(tq, tk, tv, tdo, a, sl2);
  if (cudaGetLastError() != cudaSuccess) return 31;
  return 0;
}

}  // namespace ab

// wide: 128 query rows per CTA (two warpgroups sharing the K/V ring); narrow: 64 rows, twice the CTAs
extern "C" int ab_attention_fwd(const ab::AttnArgs* a, int wide, cudaStream_t st) {
  using namespace ab;
  if (a->D % 8 != 0 || a->D > 128 || a->D <= 0) return 1;
  if (a->D <= 64) return wide ? attn_fwd_launch<64, 2>(*a, st) : attn_fwd_launch<64, 1>(*a, st);
  return wide ? attn_fwd_launch<128, 2>(*a, st) : attn_fwd_launch<128, 1>(*a, st);
}

extern "C" int ab_attention_bwd_splits(const ab::AttnArgs* a) { return ab::bwd_splits(*a); }

extern "C" int ab_attention_bwd(const ab::AttnBwdArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->f.D % 8 != 0 || a->f.D > 128 || a->f.D <= 0) return 1;
  if (a->f.D <= 64) return attn_bwd_launch<64>(*a, st);
  return attn_bwd_launch<128>(*a, st);
}
