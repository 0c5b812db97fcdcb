// Causal flash-attention forward of query chunks whose keys live in the paged bf16 KV cache (prefix caching: a short
// uncached suffix attending to a long cached prefix).
//
// The structure is the forward kernel of attention_sm90.cu: one warpgroup per 64 query rows, 64-key K/V tiles in a
// two-stage mbarrier ring, S = Q K^T with SS wgmma, grouped-query attention through kv_head = h / group, and the same
// online-softmax step and O += P V (fwd_softmax_pv in attention_sm90.cuh).  What differs is the mask (causal by
// position in the sequence), the output stores, and where a K/V tile comes from: key j of chunk c lives in cache
// row (bt[c][j >> log2 bs] << log2 bs) | (j & (bs - 1)), so a 64-key tile is one TMA box of 64 rows of one block when
// bs >= 64, or 64 / bs boxes of bs rows when bs is 16 or 32.  Every box lands at a multiple of 1024 bytes of the tile
// (bs >= 16 rows of 128 bytes), so the 128-byte swizzle of the pieces equals that of one 64-row box.
//
// Rows past the sequence's last key (the unused rows of its last block, or whole blocks it does not own when bs < 64)
// can hold anything, NaN included, and 0 * NaN in P V is NaN.  A box of a block past the sequence's last one is never
// issued (it would also read table padding), and after the last tile lands the warpgroup zeroes its rows past the
// last key in shared memory before any wgmma reads them.
//
// Grid: x = (query tile slot) * group + head within the group, y = K/V head.  The host knows only the token count T
// and the number of chunks N, so it launches (T + 63 N) / 64 tile slots, an upper bound of sum_c ceil(len_c / 64);
// each CTA finds its chunk by a warp-wide prefix sum over the chunks' tile counts and CTAs past the last tile exit.
// No atomics, no host synchronisation: the output is the same from run to run.
#include "kernels.h"
#include "attention_sm90.cuh"
#include "tma_host.h"

namespace ab {

template <int DP>
struct PagedPrefillSmem {
  static constexpr int kQ = (DP / 64) * kAtomRows64;
  static constexpr int kKV = (DP / 64) * kAtomRows64;  // one K or V tile
  static constexpr int kTotal = kQ + 4 * kKV + 64 + 1024;
};

// Chunk and tile-within-chunk of tile slot `slot`, or chunk -1 past the last tile.  Every lane of the warp returns
// the same answer.
__device__ __forceinline__ int2 find_tile(const int* __restrict__ len, int n, int slot) {
  const int lane = threadIdx.x & 31;
  int before = 0;  // tiles of the chunks already passed
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int c = c0 + lane;
    const int tiles = c < n ? (len[c] + kTile - 1) / kTile : 0;
    int incl = tiles;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, before + incl > slot);
    if (hit) {
      const int l = __ffs(hit) - 1;
      const int excl = __shfl_sync(0xffffffffu, incl - tiles, l);
      return make_int2(c0 + l, slot - before - excl);
    }
    before += __shfl_sync(0xffffffffu, incl, 31);
  }
  return make_int2(-1, 0);
}

template <int DP>
__global__ void __launch_bounds__(128, 1)
paged_prefill_sm90_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                          const __grid_constant__ CUtensorMap tv, const PagedPrefillArgs a, float scale_log2) {
  using L = PagedPrefillSmem<DP>;
  const int G = a.group;
  const int slot = blockIdx.x / G, gq = blockIdx.x - slot * G;
  const int kvh = blockIdx.y, hq = kvh * G + gq;
  const int2 ct = find_tile(a.chunk_len, a.num_chunks, slot);
  if (ct.x < 0) return;
  const int c = ct.x;
  const int len = a.chunk_len[c], pos = a.chunk_pos[c];
  const int q0 = ct.y * kTile;                 // first query of this tile within the chunk
  const int qt_row = a.chunk_start[c] + q0;    // its row of q / o
  const int shift = pos + q0;                  // position of the tile's first query
  const int kv_total = pos + len;              // keys of the sequence after this chunk
  const int kv_end = min(kv_total, shift + kTile);
  const int n_tiles = (kv_end + kTile - 1) / kTile;
  const int lg = a.block_log2, bs = 1 << lg;
  const int n_blocks = (kv_total + bs - 1) >> lg;  // blocks the sequence owns; later table entries are padding
  const int* bt = a.block_table + (long long)c * a.bt_stride;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + L::kQ;  // stage s: K at sKV + 2 s kKV, V right after
  uint64_t* bar = reinterpret_cast<uint64_t*>(sKV + 4 * L::kKV);  // [0] Q, [1 + s] K/V stage s

  // K and V of keys [64 j, 64 j + 64): one box per block piece of the tile, none for blocks the sequence does not own
  auto issue_kv = [&](int j) {
    const int s = j & 1;
    uint8_t* dk = sKV + 2 * s * L::kKV;
    uint8_t* dv = dk + L::kKV;
    const int kv0 = j * kTile;
    if (bs >= kTile) {
      const int row = (bt[kv0 >> lg] << lg) | (kv0 & (bs - 1));
      mbar_expect_tx(&bar[1 + s], 2 * L::kKV);
#pragma unroll
      for (int at = 0; at < DP / 64; ++at) {
        tma_load_3d(dk + at * kAtomRows64, &tk, &bar[1 + s], at * 64, row, kvh);
        tma_load_3d(dv + at * kAtomRows64, &tv, &bar[1 + s], at * 64, row, kvh);
      }
      return;
    }
    const int b0 = kv0 >> lg, nb = min(kTile >> lg, n_blocks - b0);
    mbar_expect_tx(&bar[1 + s], 2 * (DP / 64) * nb * bs * 128);
    for (int i = 0; i < nb; ++i) {
      const int row = bt[b0 + i] << lg;
#pragma unroll
      for (int at = 0; at < DP / 64; ++at) {
        tma_load_3d(dk + at * kAtomRows64 + i * bs * 128, &tk, &bar[1 + s], at * 64, row, kvh);
        tma_load_3d(dv + at * kAtomRows64 + i * bs * 128, &tv, &bar[1 + s], at * 64, row, kvh);
      }
    }
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(&bar[i], 1);
    mbar_fence_init();
    mbar_expect_tx(&bar[0], L::kQ);
#pragma unroll
    for (int at = 0; at < DP / 64; ++at) tma_load_4d(sQ + at * kAtomRows64, &tq, &bar[0], at * 64, qt_row, gq, kvh);
    for (int j = 0; j < 2 && j < n_tiles; ++j) issue_kv(j);
  }
  __syncthreads();

  const int tid = threadIdx.x;
  const int wi = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  float o[DP / 8][4];
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  const int row0 = wi * 16;  // first query row of this warp within the tile
  const int qpos[2] = {shift + row0 + g, shift + row0 + g + 8};
  const uint32_t q_addr = smem_u32(sQ);
  mbar_wait(&bar[0], 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j & 1;
    mbar_wait(&bar[1 + s], (j >> 1) & 1);
    const uint32_t sk = smem_u32(sKV + 2 * s * L::kKV), sv = sk + L::kKV;
    const int kv0 = j * kTile;
    if (kv0 + kTile > kv_total) {
      // the last tile of the sequence: zero K and V rows [kv_total - kv0, 64) (never loaded, or rows no one wrote)
      const int z0 = kv_total - kv0;
      const int chunks16 = (kTile - z0) * 8;  // 16-byte pieces per atom
      for (int i = tid; i < 2 * (DP / 64) * chunks16; i += 128) {
        const int atom = i / chunks16, r = i - atom * chunks16;
        sts_v4(sk + atom * kAtomRows64 + z0 * 128 + r * 16, 0u, 0u, 0u, 0u);
      }
      fence_proxy_async_smem();  // make the generic-proxy stores visible to wgmma
      __syncthreads();
    }

    float sc[8][4];  // S = Q K^T: the 16 x 64 block of this warp
    wgmma_fence();
    mma_ss_64<DP>(&sc[0][0], q_addr, kAtomRows64, sk, kAtomRows64);
    mma_sync_all();

    // scale to exp2 and mask: key j is visible to query position p iff j <= p
    const bool need_mask = kv0 + kTile - 1 > shift + row0;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[n][e] * scale_log2;
        if (need_mask && kv0 + n * 8 + 2 * t + (e & 1) > qpos[e >> 1]) v = -INFINITY;
        sc[n][e] = v;
      }
    }
    fwd_softmax_pv<DP>(sc, o, m_r, l_r, sv);
    __syncthreads();  // the warpgroup is done with stage s: refill it with tile j + 2
    if (threadIdx.x == 0 && j + 2 < n_tiles) issue_kv(j + 2);
  }

  // epilogue: O / l for the tile's rows inside the chunk
  const int H = a.kv_heads * G;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_r[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qi = q0 + row0 + g + 8 * r;
    if (qi >= len) continue;
    const float inv = l > 0.f ? 1.f / l : 0.f;
    __nv_bfloat16* og = a.o + ((long long)(qt_row + row0 + g + 8 * r) * H + hq) * DP;
#pragma unroll
    for (int dn = 0; dn < DP / 8; ++dn) {
      const int d = dn * 8 + 2 * t;
      *reinterpret_cast<uint32_t*>(og + d) = pack_bf16x2(o[dn][2 * r] * inv, o[dn][2 * r + 1] * inv);
    }
  }
}

template <int DP>
static int paged_prefill_launch(const PagedPrefillArgs& a, cudaStream_t st) {
  const int bs = 1 << a.block_log2;
  CUtensorMap tq, tk, tv;
  {
    const uint64_t dims[4] = {(uint64_t)a.D, (uint64_t)a.T, (uint64_t)a.group, (uint64_t)a.kv_heads};
    // a group of one takes the K/V-head stride for its (only ever zero) group coordinate
    const uint64_t strides[3] = {(uint64_t)a.q_stride_t, (uint64_t)(a.group > 1 ? a.q_stride_g : a.q_stride_kv),
                                 (uint64_t)a.q_stride_kv};
    if (make_tmap_bf16_4d(&tq, a.q, dims, strides, 64, kTile)) return 10;
  }
  const int box_rows = bs < kTile ? bs : kTile;
  const uint64_t row_stride = (uint64_t)a.kv_heads * a.D;
  if (make_tmap_bf16_3d(&tk, a.k_cache, a.D, a.slots, a.kv_heads, row_stride, a.D, 64, box_rows)) return 11;
  if (make_tmap_bf16_3d(&tv, a.v_cache, a.D, a.slots, a.kv_heads, row_stride, a.D, 64, box_rows)) return 12;
  auto kern = paged_prefill_sm90_kernel<DP>;
  constexpr int smem = PagedPrefillSmem<DP>::kTotal;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 20;
    attr_set = true;
  }
  const long long slots = ((long long)a.T + (long long)(kTile - 1) * a.num_chunks) / kTile;
  if (slots == 0) return 0;
  if (slots * a.group > 0x7fffffffLL) return 2;
  kern<<<dim3((unsigned)(slots * a.group), a.kv_heads), 128, smem, st>>>(tq, tk, tv, a, a.scale * 1.4426950408889634f);
  return cudaGetLastError() == cudaSuccess ? 0 : 30;
}

}  // namespace ab

extern "C" int ab_paged_prefill(const ab::PagedPrefillArgs* a, cudaStream_t st) {
  using namespace ab;
  if (a->D != 64 && a->D != 128) return 1;
  if (a->block_log2 < 4 || a->block_log2 > 10) return 3;
  return a->D == 64 ? paged_prefill_launch<64>(*a, st) : paged_prefill_launch<128>(*a, st);
}
