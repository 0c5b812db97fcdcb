// wgmma building blocks shared by the flash-attention kernels (attention_sm90.cu, paged_prefill_sm90.cu): 64-row
// tiles of 128-byte-swizzled [rows][64 head-dim elements] atoms in shared memory, the SS and RS products over them.
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

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~static_cast<uintptr_t>(1023));
}

}  // namespace ab
