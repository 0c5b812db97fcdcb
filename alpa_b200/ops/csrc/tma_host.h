// Host-side TMA tensor-map construction (driver entry point fetched through the runtime, so the
// extension does not link libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ab {

// 3-D bf16 tensor map with 128-byte swizzle used by the GEMM: dims (inner, rows, batch), strides in elements.
int make_tmap_bf16_3d(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows,
                      uint64_t batch, uint64_t row_stride_elems, uint64_t batch_stride_elems,
                      uint32_t box_inner, uint32_t box_rows);

// 4-D bf16 tensor map with 128-byte swizzle: dims (inner, rows, d2, d3), strides of dims 1..3 in elements,
// box (box_inner, box_rows, 1, 1).  Used by the attention kernels on [B, S, heads, D] views.
int make_tmap_bf16_4d(CUtensorMap* out, const void* ptr, const uint64_t* dims, const uint64_t* strides_elems,
                      uint32_t box_inner, uint32_t box_rows);

// 5-D form of the above, box (box_inner, box_rows, 1, 1, 1).  Used by the attention kernels on grouped query views
// [B, S, kv_heads, group, D] whose two head strides are not one uniform stride (the packed GQA projection).
int make_tmap_bf16_5d(CUtensorMap* out, const void* ptr, const uint64_t* dims, const uint64_t* strides_elems,
                      uint32_t box_inner, uint32_t box_rows);

int num_sms();

}  // namespace ab
