// C interface of the sm_90a bf16 GEMM (see gemm_sm90.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ab {

enum GemmAct : int {
  kActNone = 0,
  kActGelu = 1,   // out = gelu(acc + bias)
  kActRelu = 2,   // out = relu(acc + bias)
  kActDGelu = 3,  // out = acc * gelu'(aux_in)
  kActDRelu = 4,  // out = acc * (aux_in > 0)
};

constexpr int kMaxPeers = 8;

struct GemmEpilogue {
  void* out = nullptr;                     // bf16 (default) or fp32 [batch][M][ldc]
  const __nv_bfloat16* bias = nullptr;     // [N]
  const __nv_bfloat16* residual = nullptr; // [batch][M][ldc] added after activation
  __nv_bfloat16* aux_out = nullptr;        // pre-activation copy
  const __nv_bfloat16* aux_in = nullptr;   // saved pre-activation for kActDGelu/kActDRelu
  float alpha = 1.0f;
  int act = kActNone;
  int out_fp32 = 0;
  int accumulate = 0;                      // out += result
  long long ldc = 0;
  long long batch_stride_c = 0;
  int m_block_rotate = 0;                  // rotate the M-block order (staggers peer traffic)
  // fused GEMM -> reduce-scatter: row r goes to peer r / scatter_rows_per_dst, slot scatter_slot
  int scatter_rows_per_dst = 0;
  int scatter_slot = 0;
  void* scatter_ptrs[kMaxPeers] = {nullptr};
  uint32_t* scatter_flags[kMaxPeers] = {nullptr};
  // fused all-gather -> GEMM: rows of A arrive from peers; the TMA producer waits until the epoch flag of
  // the 128-row block it is about to load has been published (blocks [a_own_lo, a_own_hi) are local)
  const uint32_t* a_ready = nullptr;
  uint32_t a_ready_epoch = 0;
  int a_own_lo = 0, a_own_hi = 0;
};

struct GemmArgs {
  const void* a = nullptr;
  const void* b = nullptr;
  int M = 0, N = 0, K = 0, batch = 1;
  int a_major = 0, b_major = 0;  // 0 = K-major, 1 = MN-major
  long long lda = 0, ldb = 0;    // row stride (elements) of the stored 2-D matrix
  long long batch_stride_a = 0, batch_stride_b = 0;
  int block_n = 0;               // 0 = auto, 128 or 256
  int max_ctas = 0;              // 0 = all SMs (fused comm kernels reserve SMs)
  int epilogue_generic = 0;      // 1 = always the generic (register-store) epilogue, for comparing it with the others
  GemmEpilogue ep;
};

}  // namespace ab

extern "C" int ab_gemm_bf16(const ab::GemmArgs* g, cudaStream_t stream);
