// C interface of the non-GEMM sm_90a kernels (norm_loss_optim.cu, attention_sm90.cu, comm_sm90.cu, ...).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ab {

int num_sms();  // SMs of the current device (queried once)

struct LayerNormArgs {
  const __nv_bfloat16* x = nullptr;
  const __nv_bfloat16* residual = nullptr;  // optional: normalise (x + residual)
  const __nv_bfloat16* gamma = nullptr;
  const __nv_bfloat16* beta = nullptr;  // unused (null) when rms
  __nv_bfloat16* y = nullptr;
  __nv_bfloat16* sum_out = nullptr;  // optional: x + residual
  float* mean = nullptr;             // unused (null) when rms
  float* rstd = nullptr;
  int rows = 0, H = 0;
  float eps = 1e-5f;
  int rms = 0;  // RMSNorm: y = x * rsqrt(mean(x^2) + eps) * gamma (no mean, no beta)
};

struct LayerNormBwdArgs {
  const __nv_bfloat16* dy = nullptr;
  const __nv_bfloat16* x = nullptr;  // the normalised input (x + residual when fused)
  const __nv_bfloat16* gamma = nullptr;
  const float* mean = nullptr;          // unused (null) when rms
  const float* rstd = nullptr;
  const __nv_bfloat16* dres = nullptr;  // optional gradient flowing through the residual branch
  __nv_bfloat16* dx = nullptr;
  float* dgamma = nullptr;  // accumulated (+=)
  float* dbeta = nullptr;   // accumulated (+=); unused (null) when rms
  // [ab_layernorm_bwd_slots(rows, H)][2][H] scratch ([..][1][H] when rms): per-CTA partials of dgamma / dbeta
  float* ws = nullptr;
  int rows = 0, H = 0;
  int rms = 0;  // backward of the RMSNorm forward
};

constexpr int kMaxPeersComm = 8;
constexpr int kAdamChunk = 65536;
struct AdamTensor {
  const void* grad;
  float* master;
  float* m;
  float* v;
  __nv_bfloat16* param_bf16;  // may be null (fp32-only parameter)
  long long n;
  float weight_decay;
  int grad_is_bf16;
};
struct AdamChunk {
  int tensor;
  long long start;
};

// Grouped-query attention: query head hq = kv * group + g (g < group) attends with K/V head kv (HF's repeat_kv order);
// group == 1 is multi-head attention.
struct AttnArgs {
  const __nv_bfloat16* q = nullptr;  // [B, S, kv_heads, group, D] with arbitrary strides (elements)
  const __nv_bfloat16* k = nullptr;  // [B, S, kv_heads, D]
  const __nv_bfloat16* v = nullptr;
  __nv_bfloat16* o = nullptr;        // [B, S, kv_heads * group, D]
  float* lse = nullptr;  // [B, kv_heads * group, Sq] log-sum-exp (natural log) of scaled scores
  int B = 0, kv_heads = 0, group = 1, Sq = 0, Skv = 0, D = 0;
  long long q_stride_b = 0, q_stride_s = 0, q_stride_h = 0, q_stride_g = 0;  // q_stride_h: per K/V head
  long long k_stride_b = 0, k_stride_s = 0, k_stride_h = 0;
  long long v_stride_b = 0, v_stride_s = 0, v_stride_h = 0;
  long long o_stride_b = 0, o_stride_s = 0, o_stride_h = 0;                  // o_stride_h: per query head
  float scale = 1.f;
  int causal = 0;
  // optional device-side number of valid keys (<= Skv): lets one captured graph serve every decode position
  const int* kv_len = nullptr;
};

// Weight-streaming GEMV of the decode step (gemv_decode_sm90.cu): y[M<=8, N] = act(x[M,K] W[N,K]^T * scale + bias) + res
struct GemvArgs {
  const __nv_bfloat16* x = nullptr;
  const void* w = nullptr;               // [N, K] e4m3 (fp8 = 1) or bf16
  const float* w_scale = nullptr;        // [N] per-output-channel scale (fp8) or null
  const __nv_bfloat16* bias = nullptr;
  const __nv_bfloat16* residual = nullptr;
  __nv_bfloat16* y = nullptr;
  int M = 0, N = 0, K = 0, fp8 = 0, act = 0;
  long long ldx = 0, ldr = 0, ldy = 0;
  // optional layer norm of x on the way in (both null = none): gamma / beta [K] bf16
  const __nv_bfloat16* ln_gamma = nullptr;
  const __nv_bfloat16* ln_beta = nullptr;
  float ln_eps = 1e-5f;
  int ln_rms = 0;  // RMSNorm prologue instead (ln_beta null): y = x * rsqrt(mean(x^2) + eps) * gamma
};

struct AttnBwdArgs {
  AttnArgs f;                          // q,k,v,o,lse + shapes/strides/scale/causal of the forward
  const __nv_bfloat16* d_o = nullptr;  // [B,S,kv_heads*group,D], same strides as o
  __nv_bfloat16* dk = nullptr;         // [B,Skv,kv_heads,D]
  __nv_bfloat16* dv = nullptr;
  float* delta = nullptr;              // [B,kv_heads*group,Sq] scratch: rowsum(dO * O)
  // output strides in elements (b, s, h[, g]); D contiguous.  Lets dq/dk/dv be views of one packed
  // [B,S,h,3,D] (or [B,S,kv_heads,group+2,D]) gradient buffer so the fused-QKV dgrad/wgrad GEMMs read it without a copy.
  long long dq_stride_b = 0, dq_stride_s = 0, dq_stride_h = 0, dq_stride_g = 0;
  long long dk_stride_b = 0, dk_stride_s = 0, dk_stride_h = 0;
  long long dv_stride_b = 0, dv_stride_s = 0, dv_stride_h = 0;
  __nv_bfloat16* dq = nullptr;
  // group split of the dK / dV kernel (ab_attention_bwd_splits): splits > 1 needs ws, fp32 [2][splits][B][kv_heads][Skv][D]
  int splits = 1;
  float* ws = nullptr;
};

// Ragged 1-D token batch over a slot-addressed KV cache (serving with iteration-level batching).
struct RaggedAttnArgs {
  const __nv_bfloat16* q = nullptr;        // [T, heads, D], strides in elements, D contiguous
  const void* k_cache = nullptr;           // [slots, heads, D] bf16 or e4m3 (cache_fp8), heads*D contiguous in a row
  const void* v_cache = nullptr;
  __nv_bfloat16* o = nullptr;              // [T, heads, D]
  const int* seq_start = nullptr;          // [T] first cache row of the token's sequence (paged: its block table row)
  const int* ctx_len = nullptr;            // [T] rows attended (0 = padding token)
  const float* alibi = nullptr;            // optional [heads] slopes: score += slope * key_position
  int T = 0, heads = 0, D = 0, max_ctx = 0;
  long long q_stride_t = 0, q_stride_h = 0, o_stride_t = 0, kv_stride_s = 0;
  float scale = 1.f;
  int group = 1;  // grouped-query attention: query head h reads cache head h / group of a [slots, heads / group, D] cache
  // fp8 cache (kv_fp8.cuh): e4m3 rows, the scale of (row r, cache head h) at k/v_scale[h * scale_stride_h + r]
  int cache_fp8 = 0;
  const float* k_scale = nullptr;
  const float* v_scale = nullptr;
  long long scale_stride_h = 0;
  // Paged cache (block_table != nullptr): [N, bt_stride] int32 block ids, block size 1 << block_log2 (0..10) rows.  Key
  // j of token t lives in row (bt[seq_start[t]][j >> block_log2] << block_log2) | (j & (block size - 1)); for fp8 the
  // scales are indexed by that row too.  Entries are trusted like seq_start: the block allocator builds them, and
  // every entry a token reads (j < ctx_len) must name a block inside the cache.
  const int* block_table = nullptr;
  long long bt_stride = 0;
  int block_log2 = 0;
};

// Causal prefill of query chunks against a paged bf16 cache (paged_prefill_sm90.cu).  Chunk c is queries
// [chunk_start[c], chunk_start[c] + chunk_len[c]) of q; query i of it sits at position chunk_pos[c] + i of the sequence
// whose block table row is c, and sees that sequence's keys j <= chunk_pos[c] + i.  Key j lives in cache row
// (bt[c][j >> block_log2] << block_log2) | (j & (block size - 1)), block size 16..1024.
struct PagedPrefillArgs {
  const __nv_bfloat16* q = nullptr;     // [T, kv_heads, group, D] view: query head kv * group + g
  const __nv_bfloat16* k_cache = nullptr;  // [slots, kv_heads, D], rows dense
  const __nv_bfloat16* v_cache = nullptr;
  __nv_bfloat16* o = nullptr;           // [T, kv_heads * group, D] contiguous
  const int* chunk_start = nullptr;     // [num_chunks] each
  const int* chunk_len = nullptr;
  const int* chunk_pos = nullptr;
  const int* block_table = nullptr;     // [num_chunks, bt_stride] int32, entries trusted (the block allocator builds them)
  long long bt_stride = 0;
  long long q_stride_t = 0, q_stride_kv = 0, q_stride_g = 0;
  int T = 0, kv_heads = 0, group = 1, D = 0, slots = 0, num_chunks = 0, block_log2 = 4;
  float scale = 1.f;
};

// Decode-step attention with fused KV-cache append (decode_attention_sm90.cu).  Grouped-query attention: query head
// kv * group + g (g < group) attends with K/V head kv (HF's repeat_kv order); group == 1 is multi-head attention.
// A CTA serves a chunk of up to 8 query heads of one K/V head (ab_decode_attention_rows: the CTA rows per sequence).
struct DecodeAttnArgs {
  const __nv_bfloat16* q = nullptr;        // [B, kv_heads, group, D] view, D contiguous
  const __nv_bfloat16* k_new = nullptr;    // [B, kv_heads, D] views with one stride pair
  const __nv_bfloat16* v_new = nullptr;
  void* k_cache = nullptr;                 // [B, S_max, kv_heads, D] bf16 or e4m3 (cache_fp8), kv_heads*D dense in a row
  void* v_cache = nullptr;
  __nv_bfloat16* o = nullptr;              // [B, heads, D] contiguous, heads = kv_heads * group
  const int* kv_len = nullptr;             // device scalar: valid rows including the new one
  float* ws = nullptr;                     // [B, rows, splits, chunk, D + 2] fp32 partials (splits > 1)
  int* counters = nullptr;                 // [B * rows] arrival counters, zero between launches
  int B = 0, heads = 0, D = 0, S_max = 0, splits = 1;
  long long q_stride_b = 0, q_stride_h = 0, new_stride_b = 0, new_stride_h = 0, cache_stride_b = 0, cache_stride_s = 0;
  float scale = 1.f;
  int kv_heads = 0, group = 1;
  long long q_stride_g = 0;                // between the query heads of one K/V head
  // optional fused rotary embedding (HF's rotate_half) of the query heads and k_new before they are used:
  // pos [B] int64 positions, inv_freq [D / 2] fp32; both null = none
  const int64_t* pos = nullptr;
  const float* inv_freq = nullptr;
  // fp8 cache (kv_fp8.cuh): e4m3 rows, the scale of (sequence b, K/V head h, row s) at
  // k/v_scale[b * scale_stride_b + h * scale_stride_h + s]; the appended row is quantised in the kernel
  int cache_fp8 = 0;
  float* k_scale = nullptr;
  float* v_scale = nullptr;
  long long scale_stride_b = 0, scale_stride_h = 0;
};

// Multi-LoRA shrink / expand over segments of a ragged token batch (lora_sm90.cu).  Segment s is batch rows
// rows[seg_start[s] .. seg_start[s + 1]) and uses adapter slot seg_slot[s]; rows, seg_start and seg_slot are trusted
// like the block table (the batch assembly builds them).  A row of x / out that no segment lists is never touched.
constexpr int kLoraMaxRank = 192;  // R: up to three stacked projections of rank 64
struct LoraArgs {
  const __nv_bfloat16* x = nullptr;      // shrink input [*, K], row stride ldx
  const __nv_bfloat16* w = nullptr;      // shrink: A [slots, R, K]; expand: B [slots, N, R]
  float* y = nullptr;                    // [splits, Tl, R] fp32: shrink writes split p's partial, expand sums them
  __nv_bfloat16* out = nullptr;          // expand: [*, N], row stride ldo, updated in place
  const float* scale = nullptr;          // expand: [slots]
  const int* rows = nullptr;             // [Tl]
  const int* seg_start = nullptr;        // [S + 1]
  const int* seg_slot = nullptr;         // [S]
  long long ldx = 0, ldo = 0;
  int Tl = 0, S = 0, K = 0, N = 0, R = 0, splits = 1;
};

// Quantising store of bf16 K / V rows into an fp8 cache (kv_cache_sm90.cu).  Source token (b, t) of head h is at
// k + b * k_stride[0] + t * k_stride[1] + h * k_stride[2] (v with v_stride; D contiguous); it goes to cache row
// rows[b * T + t], or b * S + start + t when rows is null.  Cache row r of head h: data at (r * H + h) * D, scale at
// (r / S) * scale_stride_b + h * scale_stride_h + r % S.  A row outside [0, cache_rows) is not written.
struct KVStoreArgs {
  const __nv_bfloat16* k = nullptr;
  const __nv_bfloat16* v = nullptr;
  long long k_stride[3] = {0, 0, 0}, v_stride[3] = {0, 0, 0};
  uint8_t* k_data = nullptr;
  uint8_t* v_data = nullptr;
  float* k_scale = nullptr;
  float* v_scale = nullptr;
  long long scale_stride_b = 0, scale_stride_h = 0;
  const int64_t* rows = nullptr;
  int B = 0, T = 0, H = 0, D = 0, S = 0, start = 0;
  long long cache_rows = 0;
};

// Sharding-invariant counter-based dropout (dropout_sm90.cu)
constexpr int kDropoutMaxDims = 6;
struct DropoutArgs {
  const void* x = nullptr;
  void* y = nullptr;
  const unsigned long long* seed = nullptr;    // device scalar (int64 tensor)
  long long numel = 0;
  int ndim = 0;
  long long local_shape[kDropoutMaxDims] = {1, 1, 1, 1, 1, 1};
  long long offset[kDropoutMaxDims] = {0, 0, 0, 0, 0, 0};          // first global coordinate of this shard
  long long global_stride[kDropoutMaxDims] = {0, 0, 0, 0, 0, 0};   // row-major strides of the GLOBAL tensor
  uint32_t stream = 0;       // distinguishes the dropout sites of one step
  uint32_t threshold = 0;    // keep iff random word >= threshold  (= p * 2^32)
  float scale = 1.f;         // 1 / (1 - p)
};

}  // namespace ab

namespace ab {
// Base pointers of an expert buffer [E_local, G_total*C, M] on every expert-parallel peer (one entry = local).
struct MoePeers {
  void* ptr[kMaxPeersComm] = {nullptr};
  int experts_per_peer = 0;
};
}  // namespace ab

// ---- cross-mesh resharding pack / unpack (pack_sm90.cu)
namespace ab {
constexpr int kMaxPackTiles = 32;
struct PackTile {
  char* strided;            // the slice inside the stage output (source of a pack, destination of an unpack)
  char* packed;             // its position inside the contiguous staging buffer
  long long shape[4];       // box; shape[3] = BYTES of the contiguous innermost run
  long long stride[3];      // byte strides of the three outer dims of the strided side
  int vec16;                // 1 = innermost run, every stride and both addresses are multiples of 16 bytes
};
struct PackArgs {
  PackTile tiles[kMaxPackTiles];
  int num_tiles;
};
}  // namespace ab

extern "C" {
int ab_attention_fwd(const ab::AttnArgs* a, int wide, cudaStream_t st);  // wide: 128-query tiles, else 64
int ab_attention_bwd(const ab::AttnBwdArgs* a, cudaStream_t st);
int ab_attention_bwd_splits(const ab::AttnArgs* a);  // parts the dK / dV kernel splits each query-head group into
int ab_gemv_decode(const ab::GemvArgs* a, cudaStream_t st);
int ab_ragged_attention(const ab::RaggedAttnArgs* a, cudaStream_t st);
int ab_paged_prefill(const ab::PagedPrefillArgs* a, cudaStream_t st);
int ab_lora_splits(const ab::LoraArgs* a);  // K splits of the shrink for these shapes (the partials' first dim)
int ab_lora_shrink(const ab::LoraArgs* a, cudaStream_t st);
int ab_lora_expand(const ab::LoraArgs* a, cudaStream_t st);
int ab_decode_attention(const ab::DecodeAttnArgs* a, cudaStream_t st);
int ab_decode_attention_rows(const ab::DecodeAttnArgs* a);  // CTA rows per sequence (kv_heads * group chunks)
int ab_decode_attention_chunk(const ab::DecodeAttnArgs* a);  // query heads per CTA (partials per row and split)
int ab_kv_cache_store(const ab::KVStoreArgs* a, cudaStream_t st);
// out [B, end, H, D] bf16 = rows [0, end) of an fp8 cache [B, S, H, D] (data_stride_b = S * H * D), dequantised
int ab_kv_cache_load(const uint8_t* data, const float* scale, __nv_bfloat16* out, int B, int end, int H, int D,
                     long long data_stride_b, long long scale_stride_b, long long scale_stride_h, cudaStream_t st);
int ab_dropout(const ab::DropoutArgs* a, int is_bf16, cudaStream_t st);
int ab_rs_reduce(const __nv_bfloat16* staging, const uint32_t* flags, uint32_t expected, __nv_bfloat16* out,
                 const __nv_bfloat16* bias, const __nv_bfloat16* residual, int rows, int N, int tp,
                 long long slot_stride, cudaStream_t st);
int ab_ag_push(const __nv_bfloat16* src, void* const* peer_data, uint32_t* const* peer_flags, int rows, int K,
               int rank, int tp, uint32_t epoch, int include_self, cudaStream_t st);
int ab_allreduce_multimem(__nv_bfloat16* mc, long long numel, int rank, int tp, int ctas, cudaStream_t st);
int ab_peer_barrier(uint32_t* const* peer_flags, int rank, int tp, uint32_t epoch, cudaStream_t st);
int ab_allreduce_oneshot(const __nv_bfloat16* x, __nv_bfloat16* sym_local, const __nv_bfloat16* mc, long long half_stride,
                         __nv_bfloat16* out, const __nv_bfloat16* residual, long long numel, uint32_t* const* peer_flags,
                         uint32_t* counter, int rank, int tp, cudaStream_t st);
int ab_peer_barrier_auto(uint32_t* const* peer_flags, uint32_t* counter, int rank, int tp, cudaStream_t st);
int ab_layernorm_fwd(const ab::LayerNormArgs* a, cudaStream_t st);
int ab_layernorm_bwd(const ab::LayerNormBwdArgs* a, cudaStream_t st);
int ab_layernorm_bwd_slots(int rows, int H);
// x / y: [tokens, heads, D] contiguous, heads = Hkv * slots; the last slot of every K/V head (V) is copied unrotated
int ab_rotary_packed(const __nv_bfloat16* x, __nv_bfloat16* y, const int64_t* pos, const float* inv_freq, int tokens,
                     int heads, int slots, int D, int inverse, cudaStream_t st);
// gu: [pairs, 2] (gate, up); h / dh: [pairs]
int ab_swiglu_fwd(const __nv_bfloat16* gu, __nv_bfloat16* h, long long pairs, cudaStream_t st);
int ab_swiglu_bwd(const __nv_bfloat16* dh, const __nv_bfloat16* gu, __nv_bfloat16* dgu, long long pairs,
                  cudaStream_t st);
int ab_ce_stats(const __nv_bfloat16* logits, const int64_t* labels, float* stats, int rows, int V,
                int vocab_start, long long ld, cudaStream_t st);
int ab_ce_grad(__nv_bfloat16* logits, const int64_t* labels, const float* gstats,
               const float* row_scale, int rows, int V, int vocab_start, long long ld,
               cudaStream_t st);
int ab_embedding_fwd(const int64_t* ids, const int64_t* pos, const __nv_bfloat16* wte,
                     const __nv_bfloat16* wpe, __nv_bfloat16* out, int T, int H, int vocab_start,
                     int Vlocal, cudaStream_t st);
// sorted_ids / order: the token ids sorted stably by value and the token index at each sorted position
int ab_embedding_bwd(const int64_t* sorted_ids, const int64_t* order, const __nv_bfloat16* dy, float* dtable, int T,
                     int H, int vocab_start, int Vlocal, cudaStream_t st);
// ws: [ab_colsum_slots(M, N)][N] fp32 scratch
int ab_colsum_slots(int M, int N);
int ab_colsum(const __nv_bfloat16* x, float* out, float* ws, int M, int N, long long ld, cudaStream_t st);
int ab_adamw(const ab::AdamTensor* tensors, const ab::AdamChunk* chunks, int num_chunks, float lr,
             float beta1, float beta2, float eps, float bc1, float bc2, float grad_scale,
             const float* clip_coef, const float* step_ptr, cudaStream_t st);
int ab_moe_top2_route(const float* gates, int64_t* expert, int64_t* slot, int G, int S, int E, int C,
                      cudaStream_t st);
int ab_moe_dispatch(const __nv_bfloat16* x, const int64_t* expert, const int64_t* slot, const __nv_bfloat16* weight,
                    const ab::MoePeers* dst, int G, int S, int K, int M, int C, int g_off, int G_total,
                    cudaStream_t st);
int ab_moe_combine(const ab::MoePeers* src, const int64_t* expert, const int64_t* slot, const __nv_bfloat16* weight,
                   __nv_bfloat16* out, int G, int S, int K, int M, int C, int g_off, int G_total, cudaStream_t st);
int ab_moe_combine_wgrad(const __nv_bfloat16* dout, const ab::MoePeers* src, const int64_t* expert,
                         const int64_t* slot, __nv_bfloat16* dw, int G, int S, int K, int M, int C, int g_off,
                         int G_total, cudaStream_t st);
int ab_quantize_rows_e4m3(const __nv_bfloat16* x, uint8_t* q, float* scale, int M, int K, long long ldx,
                          cudaStream_t st);
int ab_gemm_fp8(const uint8_t* a, const uint8_t* b, const float* sx, const float* sw, const __nv_bfloat16* bias,
                __nv_bfloat16* out, int M, int N, int K, long long ldc, int act, cudaStream_t st);
int ab_pack_tiles(const ab::PackArgs* args, int unpack, cudaStream_t st);
int ab_quantize_rows_mxfp8(const __nv_bfloat16* x, uint8_t* q, uint8_t* sf, int M, int K, long long ldx, cudaStream_t st);
int ab_gemm_mxfp8(const uint8_t* a, const uint8_t* sfa, const uint8_t* b, const uint8_t* sfb, const __nv_bfloat16* bias,
                  __nv_bfloat16* out, int M, int N, int K, long long ldc, int act, cudaStream_t st);
// ws: [ab_sumsq_slots(num_chunks)] fp32 scratch
int ab_sumsq_slots(int num_chunks);
int ab_sumsq(const ab::AdamTensor* tensors, const ab::AdamChunk* chunks, int num_chunks, float* out, float* ws,
             cudaStream_t st);
}
