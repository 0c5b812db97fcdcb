// alpa_b200 GEMMs for sm_90a: persistent, warp-specialised, TMA -> smem ring -> wgmma.mma_async (accumulators in the
// registers of two consumer warpgroups) -> epilogue (bf16: staged in shared memory and TMA-stored for the training
// step's epilogue kinds, register stores for everything else; see kEpi*).
//
// Replaces the reference's cuBLAS custom-call path (XLA/service/gpu/matmul_utils.cc:438-480) for
// K1/K3/K4/K5/K8/K13 of SURVEY.md §2.5.
//
//   bf16 : C[b, m, n] = epi( sum_k A[b, m, k] * B[b, n, k] )  (bias / GELU / residual / dGELU / fp32 accumulate /
//          peer-memory scatter).  All four operand-major combinations are supported (wgmma transposes bf16 operands
//          read from shared memory), so the backward GEMMs (dgrad: B is MN-major, wgrad: A and B are MN-major) never
//          need a transpose pass.
//            A_MAJOR == K : A stored [batch][M][K] (K contiguous)     A_MAJOR == MN : stored [batch][K][M]
//            B_MAJOR == K : B stored [batch][N][K] (K contiguous)     B_MAJOR == MN : stored [batch][K][N]
//   fp8  : y[M,N] = act((xq[M,K] . wq[N,K]^T) * sx[m] * sw[n] + bias[n]), e4m3 operands (serving path).  Weights carry one
//          fp32 scale per output channel; activations are quantised per token on the fly by `quantize_rows_e4m3_kernel`.
//   mxfp8: OCP microscaling, e4m3 elements with one UE8M0 scale per 32 consecutive K elements.  Hopper's tensor cores
//          have no block scaling, so every K = 32 wgmma (exactly one scale block) goes to a scratch accumulator that is
//          folded into the result with both scales in registers.
//
// Block: 384 threads.  Warpgroup 0 = TMA producer (one thread issues), warpgroups 1 and 2 = consumers, each owning 64
// of the 128 rows of a tile.  Shared-memory tiles are 128-byte rows (64 bf16 or 128 e4m3 of K) with 128-byte swizzle;
// the smem descriptors below follow the canonical GMMA layouts (cute/atom/mma_traits_sm90_gmma.hpp).
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>

#include "gemm_sm90.h"
#include "kernels.h"
#include "ptx.cuh"
#include "tma_host.h"
#include "wgmma.cuh"

namespace ab {

constexpr int BLOCK_M = 128;
constexpr int kRowBytes = 128;  // K bytes per stage: 64 bf16 or 128 e4m3
constexpr int kNumThreads = 384;
constexpr int kGroupM = 16;  // M-blocks per band of the tile order (see tile_coords)

enum : uint32_t { kMajorK = 0, kMajorMN = 1 };  // operand major (wgmma transpose flag)
enum : int { kModeBf16 = 0, kModeFp8 = 1, kModeMx = 2 };

// bf16 epilogue kinds.  Each is its own instantiation, so the fully unrolled fragment loop holds only the work of one
// kind.  The fast kinds (all but kEpiGeneric) stage the bf16 tile in shared memory and write it with TMA stores; they
// need alpha == 1, a bf16 output without accumulate or residual, and output / aux tensors a TMA map can describe.
// kEpiGeneric keeps every runtime option (alpha, residual, fp32 output, accumulate, peer scatter, odd row strides)
// and stores from registers.
enum : int {
  kEpiGeneric = 0,
  kEpiStore = 1,        // out = acc
  kEpiBias = 2,         // out = acc + bias
  kEpiBiasGeluAux = 3,  // aux_out = acc + bias, out = gelu(aux_out)
  kEpiDGelu = 4,        // out = acc * gelu'(aux_in)
};

template <int BLOCK_N, int EPI>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * kRowBytes;  // 16 KB
  static constexpr int kBBytes = BLOCK_N * kRowBytes;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (BLOCK_N == 256) ? 4 : 6;
  // Fast epilogue kinds: each consumer warpgroup owns two 64 x 64 bf16 chunk buffers (128-byte rows, 128-byte
  // swizzle), so it fills one while the TMA store of the other reads it, and a copy of the tile's bias slice.  The
  // generic epilogue reserves neither: shared memory it does not use is left to the L1 cache, which the fp8 and
  // MXFP8 epilogues read their scales through.
  static constexpr int kChunkBytes = 64 * 64 * 2;
  static constexpr int kStagingBytes = EPI == kEpiGeneric ? 0 : 2 * 2 * kChunkBytes;
  static constexpr int kBiasBytes = EPI == kEpiGeneric ? 0 : 2 * BLOCK_N * 2;
  static constexpr int kTotal = kStages * kStageBytes + kStagingBytes + 1024 /*barriers*/ + kBiasBytes +
                                1024 /*align slack*/;
  static_assert(kTotal <= 232448, "exceeds the 227 KB of shared memory per block");
};

// fp8 / mxfp8 epilogue and scale operands
struct Fp8Params {
  const float* sx = nullptr;     // fp8: [M] per-row scale
  const float* sw = nullptr;     // fp8: [N] per-channel scale
  const uint8_t* sfa = nullptr;  // mxfp8: UE8M0 scale atoms of A (layout: quantize_rows_mxfp8_kernel)
  const uint8_t* sfb = nullptr;
  int num_k_atoms = 0;
  const __nv_bfloat16* bias = nullptr;
  __nv_bfloat16* out = nullptr;
  long long ldc = 0;
  int act = 0;
};

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N));
}
__device__ __forceinline__ void wg_barrier(int id) { asm volatile("bar.sync %0, 128;\n" ::"r"(id) : "memory"); }

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float dgelu_erf(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// UE8M0 scale of (row, 32-element K block)
__device__ __forceinline__ float mx_scale(const uint8_t* sf, int num_k_atoms, int row, int blk) {
  const int rr = row & 127;
  const uint8_t e = sf[((size_t)(row >> 7) * num_k_atoms + (blk >> 2)) * 512 + (rr & 31) * 16 + (rr >> 5) * 4 + (blk & 3)];
  return e == 0 ? ldexpf(1.f, -127) : __uint_as_float((uint32_t)e << 23);
}

// tmap_c / tmap_aux (fast epilogue kinds only): the bf16 output and aux_out or aux_in as (N, M, batch) maps with
// 64 x 64 boxes.  The extents are exact, so TMA clips the M and N tails of a tile.
template <int BLOCK_N, int MODE, uint32_t A_MAJOR, uint32_t B_MAJOR, int EPI>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_sm90_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_aux,
                 const GemmEpilogue ep, const Fp8Params fp, int M, int N, int K, int batch) {
  using L = SmemLayout<BLOCK_N, EPI>;
  constexpr int kStages = L::kStages;
  constexpr int kElemBytes = MODE == kModeBf16 ? 2 : 1;
  constexpr int kBlockK = kRowBytes / kElemBytes;
  constexpr int kMmaK = 32 / kElemBytes;  // K per wgmma: 16 bf16 / 32 e4m3 (32 bytes either way)
  static_assert(EPI == kEpiGeneric || MODE == kModeBf16, "fast epilogue kinds are bf16 only");
  constexpr bool kHasBias = EPI == kEpiBias || EPI == kEpiBiasGeluAux;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * L::kABytes;
  uint8_t* smem_out = smem + kStages * L::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_out + L::kStagingBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* aux_bar = empty_bar + kStages;  // [2 consumer warpgroups][2 chunk buffers]: aux_in loads
  uint32_t* bias_smem = reinterpret_cast<uint32_t*>(smem_out + L::kStagingBytes + 1024);  // [2][BLOCK_N / 2] pairs

  const int wg = threadIdx.x >> 7;
  const int num_m_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  const int num_n_blocks = (N + BLOCK_N - 1) / BLOCK_N;
  const int tiles_per_batch = num_m_blocks * num_n_blocks;
  const int num_tiles = tiles_per_batch * batch;
  const int num_k_blocks = (K + kBlockK - 1) / kBlockK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    if constexpr (EPI == kEpiDGelu) {
      for (int i = 0; i < 4; ++i) mbar_init(&aux_bar[i], 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  // Tile order: batch outermost, then bands of kGroupM M-blocks; inside a band consecutive tile ids walk M first, then
  // N.  The CTAs resident at one time (one tile id each) then cover about kGroupM A row-panels and
  // #SMs / kGroupM B column-panels, so both operands are fetched from DRAM about once per wave and reused from L2.
  // Walking M over the whole matrix instead would re-read all of A every wave once A outgrows the 50 MB L2, which it
  // does at training shapes (16384 tokens x K = 2048 bf16 is already 64 MB).  The last band holds the M tail.
  auto tile_coords = [&](int tile, int& b, int& m_blk, int& n_blk) {
    b = tile / tiles_per_batch;
    const int t = tile - b * tiles_per_batch;
    const int first = t / (kGroupM * num_n_blocks) * kGroupM;
    const int rows = min(kGroupM, num_m_blocks - first);
    const int r = t - first * num_n_blocks;
    n_blk = r / rows;
    m_blk = first + (r - n_blk * rows);
    if (ep.m_block_rotate) m_blk = (m_blk + ep.m_block_rotate) % num_m_blocks;
  };

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int b, m_blk, n_blk;
        tile_coords(tile, b, m_blk, n_blk);
        const int m0 = m_blk * BLOCK_M, n0 = n_blk * BLOCK_N;
        if (ep.a_ready != nullptr && (m_blk < ep.a_own_lo || m_blk >= ep.a_own_hi)) {
          // all-gather -> GEMM: wait for the peer that owns these rows to publish them (silent trap: see mbar_wait)
          uint32_t spins = 0;
          while (ld_acquire_sys(ep.a_ready + m_blk) < ep.a_ready_epoch) {
            __nanosleep(64);
            if (++spins > (1u << 24)) __trap();
          }
          asm volatile("fence.proxy.async;\n" ::: "memory");
        }
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], L::kStageBytes);
          uint8_t* sa = smem_a + stage * L::kABytes;
          uint8_t* sb = smem_b + stage * L::kBBytes;
          const int k0 = kb * kBlockK;
          if (A_MAJOR == kMajorK) {
            tma_load_3d(sa, &tmap_a, &full_bar[stage], k0, m0, b);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_3d(sa + j * (kBlockK * 128), &tmap_a, &full_bar[stage], m0 + j * 64, k0, b);
          }
          if (B_MAJOR == kMajorK) {
            tma_load_3d(sb, &tmap_b, &full_bar[stage], k0, n0, b);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_3d(sb + j * (kBlockK * 128), &tmap_b, &full_bar[stage], n0 + j * 64, k0, b);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma mainloop + epilogue =====================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;                   // rows [64 cw, 64 cw + 64) of the tile
  const int tid = threadIdx.x & 127;
  const int wi = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  uint32_t stage = 0, phase = 0;
  float acc[BLOCK_N / 2];
  // fast epilogue state of this warpgroup: its two staging buffers, its aux_in barriers and bias slice, the number
  // of TMA stores it has issued (they alternate between the buffers) and the parities of its aux_in barriers
  uint8_t* const stage_out = smem_out + cw * (2 * L::kChunkBytes);
  uint64_t* const aux_bar_wg = aux_bar + 2 * cw;
  uint32_t* const bias_wg = bias_smem + cw * (BLOCK_N / 2);
  uint32_t store_count = 0, aux_phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int b, m_blk, n_blk;
    tile_coords(tile, b, m_blk, n_blk);
    const int row_base = m_blk * BLOCK_M + cw * 64 + wi * 16 + g;  // + 8 for the second row of a fragment
    const int n0 = n_blk * BLOCK_N;
    const int m0w = m_blk * BLOCK_M + cw * 64;  // first row of this warpgroup
    const int n_chunks = m0w < M ? min(BLOCK_N / 64, (N - n0 + 63) / 64) : 0;  // 64-column chunks with data
    // Epilogue operands are fetched before the mainloop, so their latency hides behind it: the tile's bias slice by
    // cp.async into this warpgroup's copy (its readers passed the previous tile's last wg_barrier), and aux_in's first
    // two 64-column chunks by TMA into the staging buffers (once the previous tile's stores have finished reading them).
    if constexpr (kHasBias) {
      if (tid < BLOCK_N / 2 && n0 + 2 * tid < N)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(bias_wg + tid)),
                     "l"(ep.bias + n0 + 2 * tid)
                     : "memory");
    }
    if constexpr (EPI == kEpiDGelu) {
      if (tid == 0) {
        tma_store_wait_read<0>();
        for (int c = 0; c < 2 && c < n_chunks; ++c) {
          mbar_expect_tx(&aux_bar_wg[c], L::kChunkBytes);
          tma_load_3d(stage_out + c * L::kChunkBytes, &tmap_aux, &aux_bar_wg[c], n0 + 64 * c, m0w, b);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;

    float part0[MODE == kModeFp8 ? BLOCK_N / 2 : 1], part1[MODE == kModeFp8 ? BLOCK_N / 2 : 1];  // fp8 scratch
    auto fold = [&](const float* part) {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] += part[i];
    };
    uint32_t prev_stage = 0;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem_a + stage * L::kABytes) + cw * 8192;
      const uint32_t sb = smem_u32(smem_b + stage * L::kBBytes);
      if constexpr (MODE == kModeBf16) {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) {
          const uint64_t da = A_MAJOR == kMajorK ? gmma_desc_sw128(sa + k * 32, 16, 1024)
                                                 : gmma_desc_sw128(sa + k * (kMmaK * 128), kBlockK * 128, 1024);
          const uint64_t db = B_MAJOR == kMajorK ? gmma_desc_sw128(sb + k * 32, 16, 1024)
                                                 : gmma_desc_sw128(sb + k * (kMmaK * 128), kBlockK * 128, 1024);
          if constexpr (BLOCK_N == 256)
            wgmma_m64n256k16_bf16<A_MAJOR, B_MAJOR>(acc, da, db, 1u);
          else
            wgmma_m64n128k16_bf16<A_MAJOR, B_MAJOR>(acc, da, db, 1u);
        }
        wgmma_commit();
        // keep one group in flight: the previous stage's MMAs are done once at most one group is pending
        wgmma_wait<1>();
        if (kb > 0 && tid == 0) mbar_arrive(&empty_bar[prev_stage]);
      } else if constexpr (MODE == kModeFp8) {
        // Hopper's fp8 wgmma accumulates with fewer mantissa bits than fp32, so one chain over all of K loses
        // precision as K grows.  Each k-block (4 wgmmas, 128 K) goes to a scratch accumulator that is added to acc
        // in fp32, as CUTLASS's sm90 fp8 mainloop promotes every 4 wgmmas.  Two scratch accumulators alternate so
        // that one group stays in flight while the previous block is added.
        auto issue = [&](float* part) {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBlockK / kMmaK; ++k)
            wgmma_m64n128k32_e4m3(part, gmma_desc_sw128(sa + k * 32, 16, 1024),
                                  gmma_desc_sw128(sb + k * 32, 16, 1024), k == 0 ? 0u : 1u);
          wgmma_commit();
          wgmma_wait<1>();
        };
        if (kb & 1) {
          issue(part1);
          fold(part0);
        } else {
          issue(part0);
          if (kb > 0) fold(part1);
        }
        if (kb > 0 && tid == 0) mbar_arrive(&empty_bar[prev_stage]);
      } else {
        // block-scaled: one K = 32 product per scale block, folded in with sa(row) * sb(col)
#pragma unroll 1
        for (int k = 0; k < kBlockK / kMmaK; ++k) {
          const int blk = kb * (kBlockK / 32) + k;
          if (blk * 32 >= K) break;
          float part[BLOCK_N / 2];
          wgmma_fence();
          wgmma_m64n128k32_e4m3(part, gmma_desc_sw128(sa + k * 32, 16, 1024), gmma_desc_sw128(sb + k * 32, 16, 1024),
                                0u);
          wgmma_commit();
          wgmma_wait<0>();
          const float s_lo = mx_scale(fp.sfa, fp.num_k_atoms, min(row_base, M - 1), blk);
          const float s_hi = mx_scale(fp.sfa, fp.num_k_atoms, min(row_base + 8, M - 1), blk);
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int col = min(n0 + j * 8 + 2 * t4, N - 2);
            const float sb0 = mx_scale(fp.sfb, fp.num_k_atoms, col, blk);
            const float sb1 = mx_scale(fp.sfb, fp.num_k_atoms, col + 1, blk);
            acc[4 * j + 0] += part[4 * j + 0] * s_lo * sb0;
            acc[4 * j + 1] += part[4 * j + 1] * s_lo * sb1;
            acc[4 * j + 2] += part[4 * j + 2] * s_hi * sb0;
            acc[4 * j + 3] += part[4 * j + 3] * s_hi * sb1;
          }
        }
        if (tid == 0) mbar_arrive(&empty_bar[stage]);
      }
      prev_stage = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    if constexpr (MODE != kModeMx) {
      wgmma_wait<0>();
      if (num_k_blocks > 0 && tid == 0) mbar_arrive(&empty_bar[prev_stage]);
    }
    if constexpr (MODE == kModeFp8) {
      if (num_k_blocks & 1)
        fold(part0);
      else
        fold(part1);
    }

    // ---- epilogue: fragment j of this thread = rows (row_base, row_base + 8), columns n0 + 8 j + 2 t4 + {0, 1}
    if constexpr (EPI != kEpiGeneric) {
      // Chunk c = columns [64 c, 64 c + 64) of the warpgroup's 64 rows.  In a 128-byte-swizzled 64 x 64 bf16 buffer,
      // element (r, col) sits at byte r * 128 + ((col / 8) ^ (r % 8)) * 16 + (col % 8) * 2; fragment row r = 16 wi +
      // g + 8 hi has r % 8 == g, and the 32 lanes of a warp hit 32 different banks.
      auto frag_off = [&](int jj, int hi) -> uint32_t {
        return (wi * 16 + g + 8 * hi) * 128 + ((jj ^ g) << 4) + t4 * 4;
      };
      if constexpr (kHasBias) {
        asm volatile("cp.async.wait_all;\n" ::: "memory");  // read after the first wg_barrier of the chunk loop
      }
      // Stage one chunk (value(j, hi) -> bf16x2 of fragment j, row half hi) and TMA-store it.  Before a buffer is
      // refilled, only the read of the store issued from it two stores earlier must be complete; the writes to
      // global memory stay in flight into the next tile's mainloop.
      auto store_chunk = [&](const CUtensorMap* map, int c, auto&& value) {
        uint8_t* buf = stage_out + (store_count & 1) * L::kChunkBytes;
        const uint32_t sbuf = smem_u32(buf);
        if (tid == 0) tma_store_wait_read<1>();
        wg_barrier(1 + cw);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int hi = 0; hi < 2; ++hi) {
            const uint32_t v = value(8 * c + jj, hi);
            asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(sbuf + frag_off(jj, hi)), "r"(v) : "memory");
          }
        }
        fence_proxy_async_smem();
        wg_barrier(1 + cw);
        if (tid == 0) {
          tma_store_3d(map, buf, n0 + 64 * c, m0w, b);
          tma_store_commit();
        }
        ++store_count;
      };
      auto biased = [&](int j, int hi) {
        const float2 f = unpack_bf16x2(bias_wg[4 * j + t4]);
        return make_float2(acc[4 * j + 2 * hi] + f.x, acc[4 * j + 2 * hi + 1] + f.y);
      };
#pragma unroll
      for (int c = 0; c < BLOCK_N / 64; ++c) {
        if (c >= n_chunks) break;
        if constexpr (EPI == kEpiStore) {
          store_chunk(&tmap_c, c, [&](int j, int hi) { return pack_bf16x2(acc[4 * j + 2 * hi], acc[4 * j + 2 * hi + 1]); });
        } else if constexpr (EPI == kEpiBias) {
          store_chunk(&tmap_c, c, [&](int j, int hi) {
            const float2 v = biased(j, hi);
            return pack_bf16x2(v.x, v.y);
          });
        } else if constexpr (EPI == kEpiBiasGeluAux) {
          // the pre-activation (saved for GELU backward) and the output, staged in one pass: one buffer each
          const uint32_t s_aux = smem_u32(stage_out), s_out = smem_u32(stage_out + L::kChunkBytes);
          if (tid == 0) tma_store_wait_read<0>();
          wg_barrier(1 + cw);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
            for (int hi = 0; hi < 2; ++hi) {
              const float2 v = biased(8 * c + jj, hi);
              asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(s_aux + frag_off(jj, hi)), "r"(pack_bf16x2(v.x, v.y))
                           : "memory");
              asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(s_out + frag_off(jj, hi)),
                           "r"(pack_bf16x2(gelu_erf(v.x), gelu_erf(v.y)))
                           : "memory");
            }
          }
          fence_proxy_async_smem();
          wg_barrier(1 + cw);
          if (tid == 0) {
            tma_store_3d(&tmap_aux, stage_out, n0 + 64 * c, m0w, b);
            tma_store_3d(&tmap_c, stage_out + L::kChunkBytes, n0 + 64 * c, m0w, b);
            tma_store_commit();
          }
        } else {
          // kEpiDGelu: chunk c's aux_in was loaded into buffer c % 2; the result overwrites it in place and is
          // stored from there.  Chunk c + 2 is then loaded into the same buffer once that store has read it.
          const int bi = c & 1;
          uint8_t* buf = stage_out + bi * L::kChunkBytes;
          const uint32_t sbuf = smem_u32(buf);
          mbar_wait(&aux_bar_wg[bi], (aux_phase >> bi) & 1);
          aux_phase ^= 1u << bi;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
            for (int hi = 0; hi < 2; ++hi) {
              const int j = 8 * c + jj;
              uint32_t zb;
              asm volatile("ld.shared.b32 %0, [%1];\n" : "=r"(zb) : "r"(sbuf + frag_off(jj, hi)) : "memory");
              const float2 z = unpack_bf16x2(zb);
              const uint32_t v = pack_bf16x2(acc[4 * j + 2 * hi] * dgelu_erf(z.x), acc[4 * j + 2 * hi + 1] * dgelu_erf(z.y));
              asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(sbuf + frag_off(jj, hi)), "r"(v) : "memory");
            }
          }
          fence_proxy_async_smem();
          wg_barrier(1 + cw);
          if (tid == 0) {
            tma_store_3d(&tmap_c, buf, n0 + 64 * c, m0w, b);
            tma_store_commit();
            if (c + 2 < n_chunks) {
              tma_store_wait_read<0>();
              mbar_expect_tx(&aux_bar_wg[bi], L::kChunkBytes);
              tma_load_3d(buf, &tmap_aux, &aux_bar_wg[bi], n0 + 64 * (c + 2), m0w, b);
            }
          }
        }
      }
    } else if constexpr (MODE == kModeBf16) {
#pragma unroll
      for (int hi = 0; hi < 2; ++hi) {
        const int row = row_base + 8 * hi;
        if (row >= M) continue;
        size_t out_off;
        uint8_t* out_base = reinterpret_cast<uint8_t*>(ep.out);
        if (ep.scatter_rows_per_dst > 0) {
          // fused GEMM -> reduce-scatter: rows are routed to the owning GPU's staging buffer over peer mappings
          const int dst = row / ep.scatter_rows_per_dst;
          const int lrow = row - dst * ep.scatter_rows_per_dst;
          out_base = reinterpret_cast<uint8_t*>(ep.scatter_ptrs[dst]);
          out_off = (static_cast<size_t>(ep.scatter_slot) * ep.scatter_rows_per_dst + lrow) * static_cast<size_t>(ep.ldc);
        } else {
          out_off = static_cast<size_t>(b) * ep.batch_stride_c + static_cast<size_t>(row) * ep.ldc;
        }
        const size_t aux_off = static_cast<size_t>(b) * ep.batch_stride_c + static_cast<size_t>(row) * ep.ldc;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = n0 + j * 8 + 2 * t4;
          if (col >= N) continue;  // N % 8 == 0: col + 1 < N whenever col < N
          float v0 = acc[4 * j + 2 * hi] * ep.alpha, v1 = acc[4 * j + 2 * hi + 1] * ep.alpha;
          if (ep.bias != nullptr) {
            const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ep.bias + col));
            v0 += f.x;
            v1 += f.y;
          }
          if (ep.aux_out != nullptr)  // save pre-activation (needed by GELU backward)
            *reinterpret_cast<uint32_t*>(ep.aux_out + aux_off + col) = pack_bf16x2(v0, v1);
          if (ep.act == kActGelu) {
            v0 = gelu_erf(v0);
            v1 = gelu_erf(v1);
          } else if (ep.act == kActRelu) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          } else if (ep.act == kActDGelu || ep.act == kActDRelu) {
            // v = grad wrt activation output; aux_in = saved pre-activation
            const float2 z = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ep.aux_in + aux_off + col));
            if (ep.act == kActDGelu) {
              v0 *= dgelu_erf(z.x);
              v1 *= dgelu_erf(z.y);
            } else {
              v0 = z.x > 0.f ? v0 : 0.f;
              v1 = z.y > 0.f ? v1 : 0.f;
            }
          }
          if (ep.residual != nullptr) {
            const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(ep.residual + aux_off + col));
            v0 += f.x;
            v1 += f.y;
          }
          if (ep.out_fp32) {
            float2* o = reinterpret_cast<float2*>(reinterpret_cast<float*>(out_base) + out_off + col);
            float2 tv = make_float2(v0, v1);
            if (ep.accumulate) {
              const float2 old = *o;
              tv.x += old.x;
              tv.y += old.y;
            }
            *o = tv;
          } else {
            uint32_t* o = reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(out_base) + out_off + col);
            if (ep.accumulate) {
              const float2 old = unpack_bf16x2(*o);
              v0 += old.x;
              v1 += old.y;
            }
            *o = pack_bf16x2(v0, v1);
          }
        }
      }
      // Fused GEMM -> reduce-scatter: publish "tile landed" to the owner GPU.  One counter per (dst, 32-row block);
      // the consumer kernel waits until it reaches #n-blocks * #src-ranks.
      if (ep.scatter_rows_per_dst > 0) {
        __threadfence_system();
        wg_barrier(1 + cw);
        if ((wi & 1) == 0 && lane == 0) {
          const int row_w = m_blk * BLOCK_M + cw * 64 + (wi >> 1) * 32;
          if (row_w < M && ep.scatter_flags[0] != nullptr) {
            const int dst = row_w / ep.scatter_rows_per_dst;
            const int lblk = (row_w - dst * ep.scatter_rows_per_dst) / 32;
            red_add_release_sys(ep.scatter_flags[dst] + lblk, 1u);
          }
        }
      }
    } else {
#pragma unroll
      for (int hi = 0; hi < 2; ++hi) {
        const int row = row_base + 8 * hi;
        if (row >= M) continue;
        const float srow = MODE == kModeFp8 ? fp.sx[row] : 1.f;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = n0 + j * 8 + 2 * t4;
          if (col >= N) continue;
          float v0 = acc[4 * j + 2 * hi], v1 = acc[4 * j + 2 * hi + 1];
          if (MODE == kModeFp8) {
            v0 *= srow * fp.sw[col];
            v1 *= srow * fp.sw[col + 1];
          }
          if (fp.bias != nullptr) {
            const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(fp.bias + col));
            v0 += f.x;
            v1 += f.y;
          }
          if (fp.act == kActGelu) {
            v0 = gelu_erf(v0);
            v1 = gelu_erf(v1);
          } else if (fp.act == kActRelu) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          *reinterpret_cast<uint32_t*>(fp.out + (size_t)row * fp.ldc + col) = pack_bf16x2(v0, v1);
        }
      }
    }
  }
  if constexpr (EPI != kEpiGeneric) {
    if (tid == 0) tma_store_wait<0>();  // the staging buffers must outlive the stores that read them
  }
}

// One warp per row: scale[m] = amax / 448, q = x / scale (e4m3, saturating).
__global__ void __launch_bounds__(256)
quantize_rows_e4m3_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scale,
                          int M, int K, long long ldx) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const __nv_bfloat16* xr = x + (size_t)row * ldx;
  float amax = 0.f;
  for (int i = lane * 8; i < K; i += 256) {
    const int4 v = ld_nc_v4(xr + i);
    const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(u[j]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float s = fmaxf(amax, 1e-8f) * (1.f / 448.f);
  const float inv = 1.f / s;
  if (lane == 0) scale[row] = s;
  uint8_t* qr = q + (size_t)row * K;
  for (int i = lane * 8; i < K; i += 256) {
    const int4 v = ld_nc_v4(xr + i);
    const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
    uint32_t o[2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(u[j]);
      const __nv_fp8x2_storage_t p = __nv_cvt_float2_to_fp8x2(make_float2(f.x * inv, f.y * inv), __NV_SATFINITE, __NV_E4M3);
      if (j & 1)
        o[j >> 1] |= (uint32_t)p << 16;
      else
        o[j >> 1] = (uint32_t)p;
    }
    *reinterpret_cast<uint2*>(qr + i) = make_uint2(o[0], o[1]);
  }
}

// One warp per row, 8 elements per lane per step; 4 adjacent lanes own one 32-element scale block.
// scale = 2^e with the smallest e such that amax / 2^e <= 448 (e4m3 max); q = x / 2^e, saturating.
// Scale-factor layout: atoms of 128 rows x 4 K-blocks = 512 bytes, byte (r, j) of an atom at (r % 32) * 16 + (r / 32) * 4
// + j; atoms of one 128-row group are contiguous along K.  Padding rows / K-blocks hold 127 (scale 1.0).
__global__ void __launch_bounds__(256)
quantize_rows_mxfp8_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf,
                           int M, int K, long long ldx, int num_k_atoms) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= M) return;                                    // whole warps leave together (one row per warp)
  const __nv_bfloat16* xr = x + (size_t)row * ldx;
  uint8_t* qr = q + (size_t)row * K;
  const int rr = row & 127;
  uint8_t* sf_row = sf + (size_t)(row >> 7) * num_k_atoms * 512 + (rr & 31) * 16 + (rr >> 5) * 4;
  for (int base = 0; base < K; base += 256) {
    const int i = base + lane * 8;
    const bool ok = i < K;                                 // K % 32 == 0: a 4-lane block is in or out as a whole
    float f[8];
    float amax = 0.f;
    if (ok) {
      const int4 v = ld_nc_v4(xr + i);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = unpack_bf16x2(u[j]);
        f[2 * j] = t.x;
        f[2 * j + 1] = t.y;
        amax = fmaxf(amax, fmaxf(fabsf(t.x), fabsf(t.y)));
      }
    }
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    if (!ok) continue;
    int e = -127;
    if (amax > 0.f && amax <= 3.4028234e38f) {               // finite and non-zero (an inf / nan block keeps e = -127)
      int ex;
      (void)frexpf(amax * (1.f / 448.f), &ex);             // amax / 448 = m * 2^ex, m in [0.5, 1)
      e = ex - 1;                                          // candidate: exact when m == 0.5
      if (ldexpf(amax, -e) > 448.f) e = ex;
      e = max(-127, min(127, e));
    }
    const float inv = ldexpf(1.f, -e);
    uint32_t o[2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_fp8x2_storage_t p =
          __nv_cvt_float2_to_fp8x2(make_float2(f[2 * j] * inv, f[2 * j + 1] * inv), __NV_SATFINITE, __NV_E4M3);
      if (j & 1)
        o[j >> 1] |= (uint32_t)p << 16;
      else
        o[j >> 1] = (uint32_t)p;
    }
    *reinterpret_cast<uint2*>(qr + i) = make_uint2(o[0], o[1]);
    if ((lane & 3) == 0) {
      const int blk = i >> 5;                              // global 32-element block index along K
      sf_row[(size_t)(blk >> 2) * 512 + (blk & 3)] = (uint8_t)(e + 127);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 3-D tensor map with 128-byte swizzle: dims (inner, rows, batch), strides in elements, box (box_inner, box_rows, 1).
static int make_tmap_3d(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes, const void* ptr, uint64_t inner,
                        uint64_t rows, uint64_t batch, uint64_t row_stride_elems, uint64_t batch_stride_elems,
                        uint32_t box_inner, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t d[3] = {inner, rows, batch};
  cuuint64_t st[2] = {row_stride_elems * elem_bytes,
                      (batch > 1 ? batch_stride_elems : rows * row_stride_elems) * elem_bytes};
  cuuint32_t bx[3] = {box_inner, box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(out, dtype, 3, const_cast<void*>(ptr), d, st, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

int make_tmap_bf16_4d(CUtensorMap* out, const void* ptr, const uint64_t* dims, const uint64_t* strides_elems,
                      uint32_t box_inner, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t st[3] = {strides_elems[0] * 2, strides_elems[1] * 2, strides_elems[2] * 2};
  cuuint32_t bx[4] = {box_inner, box_rows, 1, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), d, st, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

int make_tmap_bf16_5d(CUtensorMap* out, const void* ptr, const uint64_t* dims, const uint64_t* strides_elems,
                      uint32_t box_inner, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t d[5] = {dims[0], dims[1], dims[2], dims[3], dims[4]};
  cuuint64_t st[4] = {strides_elems[0] * 2, strides_elems[1] * 2, strides_elems[2] * 2, strides_elems[3] * 2};
  cuuint32_t bx[5] = {box_inner, box_rows, 1, 1, 1};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(ptr), d, st, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : static_cast<int>(r);
}

int make_tmap_bf16_3d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows,
                      uint64_t batch, uint64_t row_stride_elems, uint64_t batch_stride_elems,
                      uint32_t box_inner, uint32_t box_rows) {
  return make_tmap_3d(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, inner, rows, batch, row_stride_elems,
                      batch_stride_elems, box_inner, box_rows);
}

static int g_num_sms = 0;
int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return g_num_sms;
}

template <int BLOCK_N, int MODE, uint32_t A_MAJOR, uint32_t B_MAJOR, int EPI>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& taux,
                  const GemmEpilogue& ep, const Fp8Params& fp, int M, int N, int K, int batch, int max_ctas,
                  cudaStream_t stream) {
  auto kern = gemm_sm90_kernel<BLOCK_N, MODE, A_MAJOR, B_MAJOR, EPI>;
  constexpr int smem = SmemLayout<BLOCK_N, EPI>::kTotal;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
      return 300;
    attr_set = true;
  }
  const int tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + BLOCK_N - 1) / BLOCK_N) * batch;
  int grid = tiles < num_sms() ? tiles : num_sms();
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  kern<<<grid, kNumThreads, smem, stream>>>(ta, tb, tc, taux, ep, fp, M, N, K, batch);
  return cudaGetLastError() == cudaSuccess ? 0 : 400;
}

// The epilogue kind a bf16 GEMM runs with.  Only the kinds the training step uses are instantiated for each operand
// major combination: the plain store for all four, bias and bias + GELU + aux_out for the forward (K, K) and dGELU
// for the dgrad (K, MN).  Everything else takes the generic epilogue.
static int epilogue_kind(const GemmArgs& g) {
  const GemmEpilogue& e = g.ep;
  auto tma_ok = [](const void* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (g.epilogue_generic || e.scatter_rows_per_dst > 0 || e.a_ready != nullptr || e.out_fp32 || e.accumulate ||
      e.alpha != 1.0f || e.residual != nullptr || !tma_ok(e.out) || e.ldc % 8 != 0 ||
      (g.batch > 1 && e.batch_stride_c % 8 != 0))
    return kEpiGeneric;
  const bool fwd = g.a_major == kMajorK && g.b_major == kMajorK;
  const bool dgrad = g.a_major == kMajorK && g.b_major == kMajorMN;
  if (e.aux_in == nullptr && e.aux_out == nullptr) {
    if (e.act == kActNone) return e.bias == nullptr ? kEpiStore : (fwd ? kEpiBias : kEpiGeneric);
    return kEpiGeneric;
  }
  if (fwd && e.bias != nullptr && e.act == kActGelu && e.aux_in == nullptr && tma_ok(e.aux_out))
    return kEpiBiasGeluAux;
  if (dgrad && e.bias == nullptr && e.act == kActDGelu && e.aux_out == nullptr && tma_ok(e.aux_in)) return kEpiDGelu;
  return kEpiGeneric;
}

template <int BLOCK_N, uint32_t A_MAJOR, uint32_t B_MAJOR>
static int launch_bf16(const GemmArgs& g, cudaStream_t stream) {
  constexpr int BK = kRowBytes / 2;
  CUtensorMap ta, tb, tc{}, taux{};
  int rc;
  if (A_MAJOR == kMajorK)
    rc = make_tmap_bf16_3d(&ta, g.a, g.K, g.M, g.batch, g.lda, g.batch_stride_a, BK, BLOCK_M);
  else
    rc = make_tmap_bf16_3d(&ta, g.a, g.M, g.K, g.batch, g.lda, g.batch_stride_a, 64, BK);
  if (rc) return 100 + rc;
  if (B_MAJOR == kMajorK)
    rc = make_tmap_bf16_3d(&tb, g.b, g.K, g.N, g.batch, g.ldb, g.batch_stride_b, BK, BLOCK_N);
  else
    rc = make_tmap_bf16_3d(&tb, g.b, g.N, g.K, g.batch, g.ldb, g.batch_stride_b, 64, BK);
  if (rc) return 200 + rc;
  int kind = epilogue_kind(g);
  if (kind != kEpiGeneric) {
    // a layout the tensor-map encoder rejects is written by the generic epilogue instead
    const void* aux = kind == kEpiBiasGeluAux ? static_cast<const void*>(g.ep.aux_out)
                      : kind == kEpiDGelu     ? static_cast<const void*>(g.ep.aux_in)
                                              : nullptr;
    if (make_tmap_bf16_3d(&tc, g.ep.out, g.N, g.M, g.batch, g.ep.ldc, g.ep.batch_stride_c, 64, 64) ||
        (aux != nullptr && make_tmap_bf16_3d(&taux, aux, g.N, g.M, g.batch, g.ep.ldc, g.ep.batch_stride_c, 64, 64)))
      kind = kEpiGeneric;
  }
#define AB_LAUNCH(EPI)                                                                                      \
  return launch<BLOCK_N, kModeBf16, A_MAJOR, B_MAJOR, EPI>(ta, tb, tc, taux, g.ep, Fp8Params{}, g.M, g.N, g.K, \
                                                           g.batch, g.max_ctas, stream)
  constexpr bool kFwd = A_MAJOR == kMajorK && B_MAJOR == kMajorK;
  constexpr bool kDgrad = A_MAJOR == kMajorK && B_MAJOR == kMajorMN;
  if (kind == kEpiStore) AB_LAUNCH(kEpiStore);
  if constexpr (kFwd) {
    if (kind == kEpiBias) AB_LAUNCH(kEpiBias);
    if (kind == kEpiBiasGeluAux) AB_LAUNCH(kEpiBiasGeluAux);
  }
  if constexpr (kDgrad) {
    if (kind == kEpiDGelu) AB_LAUNCH(kEpiDGelu);
  }
  AB_LAUNCH(kEpiGeneric);
#undef AB_LAUNCH
}

template <int MODE>
static int launch_fp8(const uint8_t* a, const uint8_t* b, const Fp8Params& fp, int M, int N, int K, cudaStream_t st) {
  CUtensorMap ta, tb, unused{};
  if (make_tmap_3d(&ta, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, a, K, M, 1, K, 0, kRowBytes, BLOCK_M)) return 100;
  if (make_tmap_3d(&tb, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, b, K, N, 1, K, 0, kRowBytes, 128)) return 200;
  return launch<128, MODE, kMajorK, kMajorK, kEpiGeneric>(ta, tb, unused, unused, GemmEpilogue{}, fp, M, N, K, 1, 0,
                                                          st);
}

}  // namespace ab

extern "C" int ab_gemm_bf16(const ab::GemmArgs* g, cudaStream_t stream) {
  using namespace ab;
  if (g->N % 8 != 0 || g->K % 8 != 0 || g->M <= 0 || g->N <= 0 || g->K <= 0) return 1;
  // Narrow outputs use 128-wide tiles (more tiles -> better wave quantisation on the SMs).
  const long tiles256 = (long)((g->M + 127) / 128) * ((g->N + 255) / 256) * g->batch;
  const bool n128 = g->block_n == 128 || (g->block_n == 0 && (g->N <= 128 || tiles256 < num_sms()));
  const int key = (n128 ? 4 : 0) | (g->a_major << 1) | g->b_major;
  switch (key) {
    case 0: return launch_bf16<256, kMajorK, kMajorK>(*g, stream);
    case 1: return launch_bf16<256, kMajorK, kMajorMN>(*g, stream);
    case 2: return launch_bf16<256, kMajorMN, kMajorK>(*g, stream);
    case 3: return launch_bf16<256, kMajorMN, kMajorMN>(*g, stream);
    case 4: return launch_bf16<128, kMajorK, kMajorK>(*g, stream);
    case 5: return launch_bf16<128, kMajorK, kMajorMN>(*g, stream);
    case 6: return launch_bf16<128, kMajorMN, kMajorK>(*g, stream);
    case 7: return launch_bf16<128, kMajorMN, kMajorMN>(*g, stream);
  }
  return 2;
}

extern "C" int ab_quantize_rows_e4m3(const __nv_bfloat16* x, uint8_t* q, float* scale, int M, int K, long long ldx,
                                     cudaStream_t st) {
  if (K % 16 != 0) return 1;
  ab::quantize_rows_e4m3_kernel<<<(M * 32 + 255) / 256, 256, 0, st>>>(x, q, scale, M, K, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_gemm_fp8(const uint8_t* a, const uint8_t* b, const float* sx, const float* sw,
                           const __nv_bfloat16* bias, __nv_bfloat16* out, int M, int N, int K, long long ldc, int act,
                           cudaStream_t st) {
  if (K % 16 != 0 || N % 8 != 0) return 1;
  ab::Fp8Params fp;
  fp.sx = sx;
  fp.sw = sw;
  fp.bias = bias;
  fp.out = out;
  fp.ldc = ldc;
  fp.act = act;
  return ab::launch_fp8<ab::kModeFp8>(a, b, fp, M, N, K, st);
}

// sf must hold ceil(M / 128) * ceil(K / 128) atoms of 512 bytes, pre-filled with 127 (padding = scale 1.0).
extern "C" int ab_quantize_rows_mxfp8(const __nv_bfloat16* x, uint8_t* q, uint8_t* sf, int M, int K, long long ldx,
                                      cudaStream_t st) {
  if (K % 32 != 0) return 1;
  ab::quantize_rows_mxfp8_kernel<<<(M * 32 + 255) / 256, 256, 0, st>>>(x, q, sf, M, K, ldx, (K + 127) / 128);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_gemm_mxfp8(const uint8_t* a, const uint8_t* sfa, const uint8_t* b, const uint8_t* sfb,
                             const __nv_bfloat16* bias, __nv_bfloat16* out, int M, int N, int K, long long ldc, int act,
                             cudaStream_t st) {
  if (K % 32 != 0 || N % 8 != 0) return 1;
  ab::Fp8Params fp;
  fp.sfa = sfa;
  fp.sfb = sfb;
  fp.num_k_atoms = (K + 127) / 128;
  fp.bias = bias;
  fp.out = out;
  fp.ldc = ldc;
  fp.act = act;
  return ab::launch_fp8<ab::kModeMx>(a, b, fp, M, N, K, st);
}
