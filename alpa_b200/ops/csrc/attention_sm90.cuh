// wgmma building blocks shared by the flash-attention kernels (attention_sm90.cu, paged_prefill_sm90.cu): 64-row
// tiles of 128-byte-swizzled [rows][64 head-dim elements] atoms in shared memory, the SS and RS products over them,
// and the forward's per-tile online softmax with O += P V.
#pragma once
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ab {

constexpr int kTile = 64;                    // keys per K/V tile, rows per warpgroup
constexpr int kAtomRows64 = kTile * 128;     // bytes of one [64 rows][64 elements] swizzled atom

// SS: acc[64 x 64] (+)= X[64 rows, DP] . Y[64 rows, DP]^T; x / y = smem addresses of atom 0 (atoms x_stride apart)
template <int DP>
__device__ __forceinline__ void mma_ss_64(float* acc, uint32_t x, uint32_t x_stride, uint32_t y, uint32_t y_stride) {
#pragma unroll
  for (int kk = 0; kk < DP / 16; ++kk) {
    const uint32_t off = (kk & 3) * 32;
    wgmma_m64n64k16_bf16<0, 0>(acc, gmma_desc_sw128(x + (kk >> 2) * x_stride + off, 16, 1024),
                               gmma_desc_sw128(y + (kk >> 2) * y_stride + off, 16, 1024), kk > 0 ? 1u : 0u);
  }
}
// RS: acc[64 x DP] += F[64 rows, 64] . Z[64 rows, DP]; f = four k16 A fragments, z = smem address of Z's atom 0
template <int DP>
__device__ __forceinline__ void mma_rs(float* acc, const uint32_t (*f)[4], uint32_t z, uint32_t z_atom_bytes) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t db = gmma_desc_sw128(z + kk * 16 * 128, z_atom_bytes, 1024);
    if constexpr (DP == 64)
      wgmma_m64n64k16_bf16_rs<1>(acc, f[kk], db, 1u);
    else
      wgmma_m64n128k16_bf16_rs<1>(acc, f[kk], db, 1u);
  }
}
__device__ __forceinline__ void mma_sync_all() {
  wgmma_commit();
  wgmma_wait<0>();
}

// One key tile of the flash-attention forward's online softmax: sc = this warp's 16 x 64 score block, already scaled
// to the exp2 domain and masked (-inf), rows g and g + 8 (a quad of lanes shares a row).  Updates the running row max
// m_r and sum l_r, rescales O and runs O += P V with V's atom 0 at smem address sv.
template <int DP>
__device__ __forceinline__ void fwd_softmax_pv(const float (&sc)[8][4], float (&o)[DP / 8][4], float (&m_r)[2],
                                               float (&l_r)[2], uint32_t sv) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], sc[n][e]);
  float corr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float m_new = fmaxf(m_r[r], mx[r]);
    corr[r] = m_new == -INFINITY ? 1.f : ex2_approx(m_r[r] - m_new);
    m_r[r] = m_new;
    l_r[r] *= corr[r];
  }
  uint32_t pf[4][4];  // P as the register A operand of P V: k16 block kk = score columns [16 kk, 16 kk + 16)
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    float p[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float m = m_r[e >> 1];
      p[e] = m == -INFINITY ? 0.f : ex2_approx(sc[n][e] - m);
    }
    l_r[0] += p[0] + p[1];
    l_r[1] += p[2] + p[3];
    pf[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p[0], p[1]);
    pf[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(p[2], p[3]);
  }
#pragma unroll
  for (int i = 0; i < DP / 8; ++i) {
    o[i][0] *= corr[0];
    o[i][1] *= corr[0];
    o[i][2] *= corr[1];
    o[i][3] *= corr[1];
  }
  wgmma_fence();
  mma_rs<DP>(&o[0][0], pf, sv, kAtomRows64);  // O += P V
  mma_sync_all();
}

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~static_cast<uintptr_t>(1023));
}

}  // namespace ab
