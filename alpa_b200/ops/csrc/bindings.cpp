// Python bindings for the alpa_b200 sm_90a kernel library (torch tensors in, raw pointers out).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <atomic>
#include <cstdlib>
#include <string>
#include <unordered_map>
#include <vector>

#include "gemm_sm90.h"
#include "kernels.h"

namespace {

using torch::Tensor;
using OptTensor = c10::optional<Tensor>;

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

inline const __nv_bfloat16* bf16_ptr(const OptTensor& t) {
  if (!t.has_value() || !t->defined()) return nullptr;
  TORCH_CHECK(t->scalar_type() == at::kBFloat16, "expected bf16 tensor");
  return reinterpret_cast<const __nv_bfloat16*>(t->data_ptr());
}

// Number of alpa_b200 CUDA kernels launched by this process (bench.py reports it as gpu_launches).
static std::atomic<long long> g_launches{0};
#define AB_CHECK_RC(rc, what) TORCH_CHECK((rc) == 0, what, " failed with code ", (rc))

// C[b,m,n] = epi(sum_k A[b,m,k] * B[b,n,k]).
//   a: [.., M, K] (trans_a=false) or [.., K, M] (trans_a=true);  b: [.., N, K] or [.., K, N] (trans_b=true)
// Inner dim must be contiguous; row stride arbitrary (multiple of 8 elements); 2-D or 3-D.
Tensor gemm(const Tensor& a, const Tensor& b, bool trans_a, bool trans_b, const OptTensor& out_opt,
            const OptTensor& bias, const OptTensor& residual, const OptTensor& aux_out,
            const OptTensor& aux_in, int64_t act, double alpha, bool accumulate, bool out_fp32,
            int64_t block_n, const std::string& epilogue) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda(), "gemm: CUDA tensors required");
  TORCH_CHECK(epilogue == "auto" || epilogue == "generic", "gemm: epilogue must be 'auto' or 'generic'");
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm: bf16 only");
  TORCH_CHECK(a.dim() == b.dim() && (a.dim() == 2 || a.dim() == 3), "gemm: 2-D or 3-D operands");
  c10::cuda::CUDAGuard guard(a.device());
  const int nd = a.dim();
  ab::GemmArgs g;
  g.batch = nd == 3 ? (int)a.size(0) : 1;
  TORCH_CHECK(nd == 2 || b.size(0) == a.size(0), "gemm: batch mismatch");
  TORCH_CHECK(a.stride(nd - 1) == 1 && b.stride(nd - 1) == 1, "gemm: inner dim must be contiguous");
  const int64_t a_rows = a.size(nd - 2), a_cols = a.size(nd - 1);
  const int64_t b_rows = b.size(nd - 2), b_cols = b.size(nd - 1);
  g.M = (int)(trans_a ? a_cols : a_rows);
  g.K = (int)(trans_a ? a_rows : a_cols);
  g.N = (int)(trans_b ? b_cols : b_rows);
  TORCH_CHECK((trans_b ? b_rows : b_cols) == g.K, "gemm: contraction mismatch");
  g.a_major = trans_a ? 1 : 0;
  g.b_major = trans_b ? 1 : 0;
  g.lda = a.stride(nd - 2);
  g.ldb = b.stride(nd - 2);
  g.batch_stride_a = nd == 3 ? a.stride(0) : 0;
  g.batch_stride_b = nd == 3 ? b.stride(0) : 0;
  TORCH_CHECK(g.lda % 8 == 0 && g.ldb % 8 == 0, "gemm: row strides must be multiples of 8");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(a.data_ptr()) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(b.data_ptr()) & 15) == 0, "gemm: 16-byte alignment");
  g.a = a.data_ptr();
  g.b = b.data_ptr();
  g.block_n = (int)block_n;
  g.epilogue_generic = epilogue == "generic" ? 1 : 0;

  Tensor out;
  if (out_opt.has_value() && out_opt->defined()) {
    out = *out_opt;
    TORCH_CHECK(out.stride(out.dim() - 1) == 1, "gemm: out inner dim must be contiguous");
    out_fp32 = out.scalar_type() == at::kFloat;
    TORCH_CHECK(out_fp32 || out.scalar_type() == at::kBFloat16, "gemm: out must be bf16/fp32");
  } else {
    auto opts = a.options().dtype(out_fp32 ? at::kFloat : at::kBFloat16);
    out = nd == 3 ? torch::empty({g.batch, g.M, g.N}, opts) : torch::empty({g.M, g.N}, opts);
    TORCH_CHECK(!accumulate, "gemm: accumulate needs an explicit out");
  }
  TORCH_CHECK(out.size(out.dim() - 2) == g.M && out.size(out.dim() - 1) == g.N, "gemm: out shape");
  TORCH_CHECK(out.dim() == nd && (nd == 2 || out.size(0) == g.batch), "gemm: out batch");
  // the epilogue stores two adjacent columns at once: 4 bytes (bf16) or 8 bytes (fp32)
  const size_t out_align = out_fp32 ? 8 : 4;
  auto pair_aligned = [&](const Tensor& t, size_t align) {
    return reinterpret_cast<uintptr_t>(t.data_ptr()) % align == 0 && t.stride(t.dim() - 2) % 2 == 0 &&
           (t.dim() == 2 || t.stride(0) % 2 == 0);
  };
  TORCH_CHECK(pair_aligned(out, out_align), "gemm: out needs even row / batch strides and a ", out_align,
              "-byte aligned base");
  g.ep.out = out.data_ptr();
  g.ep.ldc = out.stride(out.dim() - 2);
  g.ep.batch_stride_c = out.dim() == 3 ? out.stride(0) : 0;
  g.ep.out_fp32 = out_fp32 ? 1 : 0;
  g.ep.accumulate = accumulate ? 1 : 0;
  g.ep.alpha = (float)alpha;
  g.ep.act = (int)act;
  if (bias.has_value() && bias->defined())
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() && bias->numel() == g.N &&
                    reinterpret_cast<uintptr_t>(bias->data_ptr()) % 4 == 0,
                "gemm: bias must be a contiguous, 4-byte aligned bf16 [N]");
  g.ep.bias = bf16_ptr(bias);
  auto same_layout = [&](const OptTensor& t, const char* name) {
    if (t.has_value() && t->defined()) {
      TORCH_CHECK(t->dim() == out.dim() && t->sizes() == out.sizes() && t->stride(t->dim() - 1) == 1 &&
                      t->stride(t->dim() - 2) == g.ep.ldc &&
                      (t->dim() == 2 || t->stride(0) == g.ep.batch_stride_c),
                  "gemm: ", name, " must share the output's sizes and layout");
      TORCH_CHECK(t->scalar_type() == at::kBFloat16 && pair_aligned(*t, 4), "gemm: ", name,
                  " must be bf16 with a 4-byte aligned base");
    }
  };
  same_layout(residual, "residual");
  same_layout(aux_out, "aux_out");
  same_layout(aux_in, "aux_in");
  g.ep.residual = bf16_ptr(residual);
  g.ep.aux_out = const_cast<__nv_bfloat16*>(bf16_ptr(aux_out));
  g.ep.aux_in = bf16_ptr(aux_in);
  AB_CHECK_RC(ab_gemm_bf16(&g, cur_stream()), "ab_gemm_bf16");
  g_launches += 1;
  return out;
}

// Fused GEMM -> reduce-scatter producer: partial products are written straight into the owner
// GPU's staging buffer (peer mapping) and a per-32-row arrival counter is bumped.
void gemm_scatter(const Tensor& a, const Tensor& b, bool trans_b, std::vector<int64_t> peer_ptrs,
                  std::vector<int64_t> flag_ptrs, int64_t slot, int64_t rows_per_dst, int64_t ldc,
                  int64_t m_block_rotate, int64_t max_ctas, bool trans_a) {
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16 && a.stride(1) == 1 &&
              b.stride(1) == 1, "gemm_scatter: contiguous bf16 operands");
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2, "gemm_scatter: 2-D operands");
  TORCH_CHECK(peer_ptrs.size() <= ab::kMaxPeers && peer_ptrs.size() == flag_ptrs.size());
  c10::cuda::CUDAGuard guard(a.device());
  ab::GemmArgs g;
  g.M = (int)(trans_a ? a.size(1) : a.size(0));
  g.K = (int)(trans_a ? a.size(0) : a.size(1));
  g.N = (int)(trans_b ? b.size(1) : b.size(0));
  TORCH_CHECK((trans_b ? b.size(0) : b.size(1)) == g.K, "gemm_scatter: contraction mismatch");
  g.a_major = trans_a ? 1 : 0;
  g.b_major = trans_b ? 1 : 0;
  g.lda = a.stride(0);
  g.ldb = b.stride(0);
  g.a = a.data_ptr();
  g.b = b.data_ptr();
  g.max_ctas = (int)max_ctas;
  g.block_n = 256;  // the consumer's arrival count assumes ceil(N / 256) tiles per row block
  g.ep.ldc = ldc;
  g.ep.scatter_rows_per_dst = (int)rows_per_dst;
  g.ep.scatter_slot = (int)slot;
  g.ep.m_block_rotate = (int)m_block_rotate;
  for (size_t i = 0; i < peer_ptrs.size(); ++i) {
    g.ep.scatter_ptrs[i] = reinterpret_cast<void*>(peer_ptrs[i]);
    g.ep.scatter_flags[i] = reinterpret_cast<uint32_t*>(flag_ptrs[i]);
  }
  g.ep.out = g.ep.scatter_ptrs[0];
  AB_CHECK_RC(ab_gemm_bf16(&g, cur_stream()), "ab_gemm_bf16(scatter)");
  g_launches += 1;
}


// ---- fused compute + collective helpers (peer memory over NVLink) ---------------------------------
void rs_reduce(int64_t staging_ptr, int64_t flags_ptr, int64_t expected, Tensor out, const OptTensor& bias,
               const OptTensor& residual, int64_t tp, int64_t slot_stride) {
  TORCH_CHECK(out.is_contiguous() && out.scalar_type() == at::kBFloat16 && out.dim() == 2);
  c10::cuda::CUDAGuard guard(out.device());
  AB_CHECK_RC(ab_rs_reduce(reinterpret_cast<const __nv_bfloat16*>(staging_ptr),
                           reinterpret_cast<const uint32_t*>(flags_ptr), (uint32_t)expected,
                           reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), bf16_ptr(bias), bf16_ptr(residual),
                           (int)out.size(0), (int)out.size(1), (int)tp, slot_stride, cur_stream()),
              "ab_rs_reduce");
  g_launches += 1;
}

void ag_push(const Tensor& src, std::vector<int64_t> peer_ptrs, std::vector<int64_t> flag_ptrs, int64_t rank,
             int64_t epoch, bool include_self) {
  TORCH_CHECK(src.is_contiguous() && src.scalar_type() == at::kBFloat16 && src.dim() == 2);
  c10::cuda::CUDAGuard guard(src.device());
  const int tp = (int)peer_ptrs.size();
  void* data[ab::kMaxPeersComm];
  uint32_t* flags[ab::kMaxPeersComm];
  TORCH_CHECK(tp <= ab::kMaxPeersComm && flag_ptrs.size() == peer_ptrs.size());
  for (int i = 0; i < tp; ++i) {
    data[i] = reinterpret_cast<void*>(peer_ptrs[i]);
    flags[i] = reinterpret_cast<uint32_t*>(flag_ptrs[i]);
  }
  AB_CHECK_RC(ab_ag_push(bf16_ptr(src), data, flags, (int)src.size(0), (int)src.size(1), (int)rank, tp,
                         (uint32_t)epoch, include_self ? 1 : 0, cur_stream()),
              "ab_ag_push");
  g_launches += 1;
}

// C = A_gathered @ B^T where rows of A arrive from peers (flags published by ag_push).
Tensor gemm_wait_a(const Tensor& a, const Tensor& b, bool trans_b, int64_t flags_ptr, int64_t epoch,
                   int64_t own_lo, int64_t own_hi, int64_t m_block_rotate, const OptTensor& bias,
                   const OptTensor& aux_out, int64_t act) {
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.scalar_type() == at::kBFloat16 && a.stride(1) == 1 && b.stride(1) == 1);
  c10::cuda::CUDAGuard guard(a.device());
  ab::GemmArgs g;
  g.M = (int)a.size(0);
  g.K = (int)a.size(1);
  g.N = (int)(trans_b ? b.size(1) : b.size(0));
  g.b_major = trans_b ? 1 : 0;
  g.lda = a.stride(0);
  g.ldb = b.stride(0);
  g.a = a.data_ptr();
  g.b = b.data_ptr();
  Tensor out = torch::empty({g.M, g.N}, a.options());
  g.ep.out = out.data_ptr();
  g.ep.ldc = g.N;
  g.ep.bias = bf16_ptr(bias);
  g.ep.aux_out = const_cast<__nv_bfloat16*>(bf16_ptr(aux_out));
  g.ep.act = (int)act;
  g.ep.m_block_rotate = (int)m_block_rotate;
  g.ep.a_ready = reinterpret_cast<const uint32_t*>(flags_ptr);
  g.ep.a_ready_epoch = (uint32_t)epoch;
  g.ep.a_own_lo = (int)own_lo;
  g.ep.a_own_hi = (int)own_hi;
  AB_CHECK_RC(ab_gemm_bf16(&g, cur_stream()), "ab_gemm_bf16(wait_a)");
  g_launches += 1;
  return out;
}

void allreduce_multimem(int64_t mc_ptr, int64_t numel, int64_t rank, int64_t tp, int64_t ctas) {
  AB_CHECK_RC(ab_allreduce_multimem(reinterpret_cast<__nv_bfloat16*>(mc_ptr), numel, (int)rank, (int)tp, (int)ctas,
                                    cur_stream()),
              "ab_allreduce_multimem");
  g_launches += 1;
}

void peer_barrier(std::vector<int64_t> flag_ptrs, int64_t rank, int64_t epoch) {
  uint32_t* flags[ab::kMaxPeersComm];
  const int tp = (int)flag_ptrs.size();
  TORCH_CHECK(tp <= ab::kMaxPeersComm);
  for (int i = 0; i < tp; ++i) flags[i] = reinterpret_cast<uint32_t*>(flag_ptrs[i]);
  AB_CHECK_RC(ab_peer_barrier(flags, (int)rank, tp, (uint32_t)epoch, cur_stream()), "ab_peer_barrier");
  g_launches += 1;
}

// Graph-capturable cross-GPU barrier: the epoch lives in `counter` (a 1-element int32 CUDA tensor owned by the caller).
void peer_barrier_auto(std::vector<int64_t> flag_ptrs, const Tensor& counter, int64_t rank) {
  uint32_t* flags[ab::kMaxPeersComm];
  const int tp = (int)flag_ptrs.size();
  TORCH_CHECK(tp <= ab::kMaxPeersComm);
  TORCH_CHECK(counter.is_cuda() && counter.numel() >= 1 && counter.element_size() == 4, "peer_barrier_auto: counter");
  for (int i = 0; i < tp; ++i) flags[i] = reinterpret_cast<uint32_t*>(flag_ptrs[i]);
  AB_CHECK_RC(ab_peer_barrier_auto(flags, reinterpret_cast<uint32_t*>(counter.data_ptr()), (int)rank, tp, cur_stream()),
              "ab_peer_barrier_auto");
  g_launches += 1;
}

// One-shot all-reduce of a small bf16 vector through a two-half symmetric staging buffer (see comm_sm90.cu).
void allreduce_oneshot(const Tensor& x, int64_t sym_local_ptr, int64_t mc_ptr, int64_t half_stride, Tensor out,
                       std::vector<int64_t> flag_ptrs, const Tensor& counter, int64_t rank, const OptTensor& residual) {
  uint32_t* flags[ab::kMaxPeersComm];
  const int tp = (int)flag_ptrs.size();
  TORCH_CHECK(tp <= ab::kMaxPeersComm && x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.is_contiguous() &&
              out.scalar_type() == at::kBFloat16 && out.is_contiguous() && out.numel() == x.numel(),
              "allreduce_oneshot: contiguous bf16 x / out of equal size");
  TORCH_CHECK(counter.is_cuda() && counter.element_size() == 4, "allreduce_oneshot: counter");
  for (int i = 0; i < tp; ++i) flags[i] = reinterpret_cast<uint32_t*>(flag_ptrs[i]);
  if (residual.has_value() && residual->defined())
    TORCH_CHECK(residual->scalar_type() == at::kBFloat16 && residual->is_contiguous() && residual->numel() == x.numel(),
                "allreduce_oneshot: residual must be contiguous bf16 of x's size");
  c10::cuda::CUDAGuard guard(x.device());
  AB_CHECK_RC(ab_allreduce_oneshot(bf16_ptr(x), reinterpret_cast<__nv_bfloat16*>(sym_local_ptr),
                                   reinterpret_cast<const __nv_bfloat16*>(mc_ptr), half_stride,
                                   reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), bf16_ptr(residual), x.numel(), flags,
                                   reinterpret_cast<uint32_t*>(counter.data_ptr()), (int)rank, tp, cur_stream()),
              "ab_allreduce_oneshot");
  g_launches += 1;
}

static void fill_attn_args(ab::AttnArgs& a, const Tensor& q, const Tensor& k, const Tensor& v,
                           double scale, bool causal) {
  TORCH_CHECK(q.dim() == 4 && k.dim() == 4 && v.dim() == 4, "attention: [B,S,h,D] tensors");
  TORCH_CHECK(q.scalar_type() == at::kBFloat16 && k.scalar_type() == at::kBFloat16 &&
              v.scalar_type() == at::kBFloat16, "attention: bf16 only");
  TORCH_CHECK(q.stride(3) == 1 && k.stride(3) == 1 && v.stride(3) == 1, "attention: D contiguous");
  a.q = bf16_ptr(q); a.k = bf16_ptr(k); a.v = bf16_ptr(v);
  a.B = (int)q.size(0); a.Sq = (int)q.size(1); a.heads = (int)q.size(2); a.D = (int)q.size(3);
  a.Skv = (int)k.size(1);
  TORCH_CHECK(k.size(0) == a.B && v.size(0) == a.B && k.size(2) == a.heads && v.size(2) == a.heads &&
              k.size(3) == a.D && v.size(3) == a.D && v.size(1) == a.Skv, "attention: shape mismatch");
  a.q_stride_b = q.stride(0); a.q_stride_s = q.stride(1); a.q_stride_h = q.stride(2);
  a.k_stride_b = k.stride(0); a.k_stride_s = k.stride(1); a.k_stride_h = k.stride(2);
  a.v_stride_b = v.stride(0); a.v_stride_s = v.stride(1); a.v_stride_h = v.stride(2);
  a.scale = (float)scale;
  a.causal = causal ? 1 : 0;
}

// q,k,v: [B,S,h,D] (any strides with D contiguous, e.g. views of a fused QKV projection).
std::vector<Tensor> attention_fwd(const Tensor& q, const Tensor& k, const Tensor& v, double scale,
                                  bool causal, const OptTensor& kv_len) {
  c10::cuda::CUDAGuard guard(q.device());
  ab::AttnArgs a;
  fill_attn_args(a, q, k, v, scale, causal);
  if (kv_len.has_value() && kv_len->defined()) {
    TORCH_CHECK(kv_len->is_cuda() && kv_len->scalar_type() == at::kInt && kv_len->numel() == 1,
                "attention: kv_len must be an int32 CUDA scalar");
    a.kv_len = kv_len->data_ptr<int>();
  }
  Tensor o = torch::empty({a.B, a.Sq, a.heads, a.D}, q.options());
  Tensor lse = torch::empty({a.B, a.heads, a.Sq}, q.options().dtype(at::kFloat));
  a.o = reinterpret_cast<__nv_bfloat16*>(o.data_ptr());
  a.lse = lse.data_ptr<float>();
  a.o_stride_b = o.stride(0); a.o_stride_s = o.stride(1); a.o_stride_h = o.stride(2);
  // 128-query tiles by default; ALPA_B200_ATTN_FWD=gen2 pins the 64-query-tile configuration (twice the CTAs).  The
  // kernel self-check (alpa_b200/ops/selfcheck.py) pins it when the default misbehaves on this GPU.
  static const bool narrow = [] {
    const char* e = std::getenv("ALPA_B200_ATTN_FWD");
    return e != nullptr && std::string(e) != "gen4";
  }();
  AB_CHECK_RC(ab_attention_fwd(&a, narrow ? 0 : 1, cur_stream()), "ab_attention_fwd");
  g_launches += 1;
  return {o, lse};
}

// Attention of a ragged 1-D token batch against a slot-addressed KV cache (see ragged_attention_sm90.cu).
Tensor ragged_attention(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& seq_start,
                        const Tensor& ctx_len, double scale, int64_t max_ctx, const OptTensor& alibi) {
  TORCH_CHECK(q.dim() == 3 && q.stride(2) == 1 && q.scalar_type() == at::kBFloat16, "ragged_attention: q must be bf16 [T, heads, D]");
  TORCH_CHECK(k_cache.dim() == 3 && v_cache.dim() == 3 && k_cache.scalar_type() == at::kBFloat16 &&
              v_cache.scalar_type() == at::kBFloat16, "ragged_attention: caches must be bf16 [slots, heads, D]");
  TORCH_CHECK(k_cache.stride(2) == 1 && k_cache.stride(1) == k_cache.size(2) && v_cache.strides() == k_cache.strides() &&
              v_cache.sizes() == k_cache.sizes(), "ragged_attention: cache rows must be dense");
  TORCH_CHECK(k_cache.size(1) == q.size(1) && k_cache.size(2) == q.size(2));
  TORCH_CHECK(seq_start.scalar_type() == at::kInt && ctx_len.scalar_type() == at::kInt && seq_start.is_contiguous() &&
              ctx_len.is_contiguous() && seq_start.numel() == q.size(0) && ctx_len.numel() == q.size(0) &&
              seq_start.is_cuda() && ctx_len.is_cuda(), "ragged_attention: seq_start / ctx_len must be int32 CUDA [T]");
  c10::cuda::CUDAGuard guard(q.device());
  ab::RaggedAttnArgs a;
  a.q = bf16_ptr(q);
  a.k_cache = bf16_ptr(k_cache);
  a.v_cache = bf16_ptr(v_cache);
  Tensor o = torch::empty({q.size(0), q.size(1), q.size(2)}, q.options());
  a.o = reinterpret_cast<__nv_bfloat16*>(o.data_ptr());
  a.seq_start = seq_start.data_ptr<int>();
  a.ctx_len = ctx_len.data_ptr<int>();
  if (alibi.has_value() && alibi->defined()) {
    TORCH_CHECK(alibi->scalar_type() == at::kFloat && alibi->is_contiguous() && alibi->numel() == q.size(1));
    a.alibi = alibi->data_ptr<float>();
  }
  a.T = (int)q.size(0); a.heads = (int)q.size(1); a.D = (int)q.size(2); a.max_ctx = (int)max_ctx;
  a.q_stride_t = q.stride(0); a.q_stride_h = q.stride(1); a.o_stride_t = o.stride(0);
  a.kv_stride_s = k_cache.stride(0);
  a.scale = (float)scale;
  AB_CHECK_RC(ab_ragged_attention(&a, cur_stream()), "ab_ragged_attention");
  g_launches += 1;
  return o;
}

// Sharding-invariant dropout: y = keep(seed, stream, global index) ? x / (1 - p) : 0   (dropout_sm90.cu)
Tensor dropout(const Tensor& x_in, double p, const Tensor& seed, int64_t stream, const std::vector<int64_t>& global_shape,
               const std::vector<int64_t>& offsets) {
  TORCH_CHECK(x_in.scalar_type() == at::kBFloat16 || x_in.scalar_type() == at::kFloat, "dropout: bf16 / fp32 only");
  TORCH_CHECK(seed.is_cuda() && seed.scalar_type() == at::kLong && seed.numel() == 1, "dropout: seed must be an int64 CUDA scalar");
  TORCH_CHECK(p >= 0.0 && p < 1.0, "dropout: p must be in [0, 1)");
  Tensor x = x_in.contiguous();
  const int nd = (int)x.dim();
  TORCH_CHECK(nd >= 1 && nd <= ab::kDropoutMaxDims && (int)global_shape.size() == nd && (int)offsets.size() == nd);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x);
  ab::DropoutArgs a;
  a.x = x.data_ptr();
  a.y = y.data_ptr();
  a.seed = reinterpret_cast<const unsigned long long*>(seed.data_ptr<int64_t>());
  a.numel = x.numel();
  a.ndim = nd;
  long long gs = 1;
  for (int d = nd - 1; d >= 0; --d) {
    a.local_shape[d] = x.size(d);
    a.offset[d] = offsets[d];
    a.global_stride[d] = gs;
    TORCH_CHECK(offsets[d] >= 0 && offsets[d] + x.size(d) <= global_shape[d], "dropout: shard outside the global tensor");
    gs *= global_shape[d];
  }
  a.stream = (uint32_t)stream;
  a.threshold = (uint32_t)std::min<double>(4294967295.0, std::floor(p * 4294967296.0));
  a.scale = (float)(1.0 / (1.0 - p));
  AB_CHECK_RC(ab_dropout(&a, x.scalar_type() == at::kBFloat16 ? 1 : 0, cur_stream()), "ab_dropout");
  g_launches += 1;
  return y;
}

// Backward of attention.  dq/dk/dv may be provided as (strided) views, e.g. slices of one packed
// [B,S,h,3,D] buffer; otherwise contiguous [B,S,h,D] tensors are allocated.
std::vector<Tensor> attention_bwd(const Tensor& d_o_in, const Tensor& q, const Tensor& k, const Tensor& v,
                                  const Tensor& o_in, const Tensor& lse, double scale, bool causal,
                                  const OptTensor& dq_out, const OptTensor& dk_out, const OptTensor& dv_out) {
  c10::cuda::CUDAGuard guard(q.device());
  Tensor d_o = d_o_in.contiguous();
  Tensor o = o_in.contiguous();
  ab::AttnBwdArgs a;
  fill_attn_args(a.f, q, k, v, scale, causal);
  TORCH_CHECK(lse.is_contiguous() && lse.scalar_type() == at::kFloat);
  a.f.o = const_cast<__nv_bfloat16*>(bf16_ptr(o));
  a.f.lse = const_cast<float*>(lse.data_ptr<float>());
  a.f.o_stride_b = o.stride(0); a.f.o_stride_s = o.stride(1); a.f.o_stride_h = o.stride(2);
  a.d_o = bf16_ptr(d_o);
  const int B = a.f.B, H = a.f.heads, Sq = a.f.Sq, Skv = a.f.Skv, D = a.f.D;
  Tensor delta = torch::empty({B, H, Sq}, q.options().dtype(at::kFloat));
  auto pick = [&](const OptTensor& t, int S) {
    if (t.has_value() && t->defined()) {
      TORCH_CHECK(t->dim() == 4 && t->stride(3) == 1 && t->scalar_type() == at::kBFloat16 && t->size(1) == S);
      return *t;
    }
    return torch::empty({B, S, H, D}, q.options());
  };
  Tensor dq = pick(dq_out, Sq), dk = pick(dk_out, Skv), dv = pick(dv_out, Skv);
  a.delta = delta.data_ptr<float>();
  a.dq = reinterpret_cast<__nv_bfloat16*>(dq.data_ptr());
  a.dk = reinterpret_cast<__nv_bfloat16*>(dk.data_ptr());
  a.dv = reinterpret_cast<__nv_bfloat16*>(dv.data_ptr());
  a.dq_stride_b = dq.stride(0); a.dq_stride_s = dq.stride(1); a.dq_stride_h = dq.stride(2);
  a.dk_stride_b = dk.stride(0); a.dk_stride_s = dk.stride(1); a.dk_stride_h = dk.stride(2);
  a.dv_stride_b = dv.stride(0); a.dv_stride_s = dv.stride(1); a.dv_stride_h = dv.stride(2);
  AB_CHECK_RC(ab_attention_bwd(&a, cur_stream()), "ab_attention_bwd");
  g_launches += 3;
  return {dq, dk, dv};
}

std::vector<Tensor> layernorm_fwd(const Tensor& x, const OptTensor& residual, const Tensor& gamma,
                                  const Tensor& beta, double eps, bool want_sum) {
  TORCH_CHECK(x.is_contiguous() && x.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(x.device());
  const int H = (int)x.size(-1);
  const int rows = (int)(x.numel() / H);
  Tensor y = torch::empty_like(x);
  Tensor mean = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor sum;
  ab::LayerNormArgs a;
  a.x = bf16_ptr(x);
  if (residual.has_value() && residual->defined()) {
    TORCH_CHECK(residual->is_contiguous() && residual->sizes() == x.sizes());
    a.residual = bf16_ptr(residual);
    if (want_sum) {
      sum = torch::empty_like(x);
      a.sum_out = reinterpret_cast<__nv_bfloat16*>(sum.data_ptr());
    }
  }
  a.gamma = bf16_ptr(gamma);
  a.beta = bf16_ptr(beta);
  a.y = reinterpret_cast<__nv_bfloat16*>(y.data_ptr());
  a.mean = mean.data_ptr<float>();
  a.rstd = rstd.data_ptr<float>();
  a.rows = rows;
  a.H = H;
  a.eps = (float)eps;
  AB_CHECK_RC(ab_layernorm_fwd(&a, cur_stream()), "ab_layernorm_fwd");
  g_launches += 1;
  return {y, mean, rstd, sum.defined() ? sum : Tensor()};
}

Tensor layernorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& gamma, const Tensor& mean,
                     const Tensor& rstd, const OptTensor& dres, Tensor dgamma, Tensor dbeta) {
  TORCH_CHECK(dy.is_contiguous() && x.is_contiguous());
  TORCH_CHECK(dgamma.scalar_type() == at::kFloat && dbeta.scalar_type() == at::kFloat);
  c10::cuda::CUDAGuard guard(x.device());
  const int H = (int)x.size(-1);
  Tensor dx = torch::empty_like(x);
  ab::LayerNormBwdArgs a;
  a.dy = bf16_ptr(dy);
  a.x = bf16_ptr(x);
  a.gamma = bf16_ptr(gamma);
  a.mean = mean.data_ptr<float>();
  a.rstd = rstd.data_ptr<float>();
  if (dres.has_value() && dres->defined()) {
    TORCH_CHECK(dres->is_contiguous());
    a.dres = bf16_ptr(dres);
  }
  a.dx = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr());
  a.dgamma = dgamma.data_ptr<float>();
  a.dbeta = dbeta.data_ptr<float>();
  a.rows = (int)(x.numel() / H);
  a.H = H;
  Tensor ws = torch::empty({(int64_t)ab_layernorm_bwd_slots(a.rows, H), 2, H}, x.options().dtype(at::kFloat));
  a.ws = ws.data_ptr<float>();
  AB_CHECK_RC(ab_layernorm_bwd(&a, cur_stream()), "ab_layernorm_bwd");
  g_launches += 3;   // row kernel + fixed-order reductions of dgamma and dbeta
  return dx;
}

Tensor ce_stats(const Tensor& logits, const Tensor& labels, int64_t vocab_start) {
  TORCH_CHECK(logits.dim() == 2 && logits.stride(1) == 1 && logits.scalar_type() == at::kBFloat16);
  TORCH_CHECK(labels.scalar_type() == at::kLong && labels.is_contiguous());
  c10::cuda::CUDAGuard guard(logits.device());
  Tensor stats = torch::empty({logits.size(0), 3}, logits.options().dtype(at::kFloat));
  AB_CHECK_RC(ab_ce_stats(bf16_ptr(logits), labels.data_ptr<int64_t>(), stats.data_ptr<float>(),
                          (int)logits.size(0), (int)logits.size(1), (int)vocab_start,
                          logits.stride(0), cur_stream()),
              "ab_ce_stats");
  g_launches += 1;
  return stats;
}

void ce_grad_(Tensor logits, const Tensor& labels, const Tensor& gstats, const Tensor& row_scale,
              int64_t vocab_start) {
  TORCH_CHECK(logits.dim() == 2 && logits.stride(1) == 1 && logits.scalar_type() == at::kBFloat16);
  TORCH_CHECK(gstats.is_contiguous() && gstats.scalar_type() == at::kFloat && gstats.size(1) == 2);
  TORCH_CHECK(row_scale.is_contiguous() && row_scale.scalar_type() == at::kFloat);
  c10::cuda::CUDAGuard guard(logits.device());
  AB_CHECK_RC(ab_ce_grad(reinterpret_cast<__nv_bfloat16*>(logits.data_ptr()),
                         labels.data_ptr<int64_t>(), gstats.data_ptr<float>(),
                         row_scale.data_ptr<float>(), (int)logits.size(0), (int)logits.size(1),
                         (int)vocab_start, logits.stride(0), cur_stream()),
              "ab_ce_grad");
  g_launches += 1;
}

Tensor embedding_fwd(const Tensor& ids, const OptTensor& pos, const Tensor& wte, const OptTensor& wpe,
                     int64_t vocab_start) {
  TORCH_CHECK(ids.scalar_type() == at::kLong && ids.is_contiguous() && wte.is_contiguous());
  c10::cuda::CUDAGuard guard(wte.device());
  const int T = (int)ids.numel(), H = (int)wte.size(1);
  auto shape = ids.sizes().vec();
  shape.push_back(H);
  Tensor out = torch::empty(shape, wte.options());
  const int64_t* pp = nullptr;
  if (pos.has_value() && pos->defined()) {
    TORCH_CHECK(pos->scalar_type() == at::kLong && pos->is_contiguous() && pos->numel() == T);
    pp = pos->data_ptr<int64_t>();
  }
  AB_CHECK_RC(ab_embedding_fwd(ids.data_ptr<int64_t>(), pp, bf16_ptr(wte), pp ? bf16_ptr(wpe) : nullptr,
                               reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), T, H,
                               (int)vocab_start, (int)wte.size(0), cur_stream()),
              "ab_embedding_fwd");
  g_launches += 1;
  return out;
}

void embedding_bwd_(const Tensor& ids, const Tensor& dy, Tensor dtable, int64_t vocab_start) {
  TORCH_CHECK(dtable.scalar_type() == at::kFloat && dtable.is_contiguous() && dy.is_contiguous());
  TORCH_CHECK(ids.scalar_type() == at::kLong, "embedding_bwd: int64 ids");
  c10::cuda::CUDAGuard guard(dy.device());
  // a stable sort groups equal ids in token order: the kernel sums each group without atomics (deterministic)
  auto sorted = at::sort(ids.reshape({-1}), /*stable=*/true, /*dim=*/0, /*descending=*/false);
  Tensor sorted_ids = std::get<0>(sorted).contiguous(), order = std::get<1>(sorted).contiguous();
  AB_CHECK_RC(ab_embedding_bwd(sorted_ids.data_ptr<int64_t>(), order.data_ptr<int64_t>(), bf16_ptr(dy),
                               dtable.data_ptr<float>(), (int)ids.numel(), (int)dtable.size(1), (int)vocab_start,
                               (int)dtable.size(0), cur_stream()),
              "ab_embedding_bwd");
  g_launches += 1;
}

void colsum_(const Tensor& x, Tensor out) {
  TORCH_CHECK(x.dim() == 2 && x.stride(1) == 1 && out.scalar_type() == at::kFloat);
  c10::cuda::CUDAGuard guard(x.device());
  const int M = (int)x.size(0), N = (int)x.size(1);
  if (M == 0) return;
  Tensor ws = torch::empty({(int64_t)ab_colsum_slots(M, N), N}, x.options().dtype(at::kFloat));
  AB_CHECK_RC(ab_colsum(bf16_ptr(x), out.data_ptr<float>(), ws.data_ptr<float>(), M, N, x.stride(0), cur_stream()),
              "ab_colsum");
  g_launches += 2;   // partials + fixed-order reduction
}

// Builds the device-side tensor/chunk tables for the fused optimizer. Returns (tensors, chunks).
std::vector<Tensor> adam_build_tables(const std::vector<Tensor>& grads, const std::vector<Tensor>& masters,
                                      const std::vector<Tensor>& ms, const std::vector<Tensor>& vs,
                                      const std::vector<OptTensor>& params,
                                      const std::vector<double>& weight_decays) {
  const size_t n = grads.size();
  TORCH_CHECK(masters.size() == n && ms.size() == n && vs.size() == n && params.size() == n &&
              weight_decays.size() == n);
  std::vector<ab::AdamTensor> tt(n);
  std::vector<ab::AdamChunk> cc;
  for (size_t i = 0; i < n; ++i) {
    TORCH_CHECK(grads[i].is_contiguous() && masters[i].is_contiguous() && ms[i].is_contiguous() &&
                vs[i].is_contiguous());
    TORCH_CHECK(masters[i].scalar_type() == at::kFloat && ms[i].scalar_type() == at::kFloat &&
                vs[i].scalar_type() == at::kFloat);
    tt[i].grad = grads[i].data_ptr();
    tt[i].grad_is_bf16 = grads[i].scalar_type() == at::kBFloat16;
    TORCH_CHECK(tt[i].grad_is_bf16 || grads[i].scalar_type() == at::kFloat);
    tt[i].master = masters[i].data_ptr<float>();
    tt[i].m = ms[i].data_ptr<float>();
    tt[i].v = vs[i].data_ptr<float>();
    tt[i].param_bf16 = const_cast<__nv_bfloat16*>(bf16_ptr(params[i]));
    tt[i].n = masters[i].numel();
    tt[i].weight_decay = (float)weight_decays[i];
    for (long long s = 0; s < tt[i].n; s += ab::kAdamChunk) cc.push_back({(int)i, s});
  }
  auto dev = masters[0].device();
  // pinned staging: the upload is an async copy that may be captured into a CUDA graph (the host tensors are
  // returned so the caller keeps them alive as long as the device tables)
  auto hopts = torch::dtype(torch::kUInt8).pinned_memory(true);
  Tensor t_host = torch::empty({(int64_t)(n * sizeof(ab::AdamTensor))}, hopts);
  Tensor c_host = torch::empty({(int64_t)(cc.size() * sizeof(ab::AdamChunk))}, hopts);
  memcpy(t_host.data_ptr(), tt.data(), n * sizeof(ab::AdamTensor));
  memcpy(c_host.data_ptr(), cc.data(), cc.size() * sizeof(ab::AdamChunk));
  return {t_host.to(dev, /*non_blocking=*/true), c_host.to(dev, /*non_blocking=*/true), t_host, c_host};
}

void adamw_step(const Tensor& tensors, const Tensor& chunks, double lr, double beta1, double beta2,
                double eps, int64_t step, double grad_scale, const OptTensor& clip_coef,
                const OptTensor& step_tensor) {
  c10::cuda::CUDAGuard guard(tensors.device());
  const int nchunks = (int)(chunks.numel() / sizeof(ab::AdamChunk));
  const float bc1 = 1.f - (float)std::pow(beta1, (double)step);
  const float bc2 = 1.f - (float)std::pow(beta2, (double)step);
  const float* cc = (clip_coef.has_value() && clip_coef->defined()) ? clip_coef->data_ptr<float>() : nullptr;
  AB_CHECK_RC(ab_adamw(reinterpret_cast<const ab::AdamTensor*>(tensors.data_ptr()),
                       reinterpret_cast<const ab::AdamChunk*>(chunks.data_ptr()), nchunks, (float)lr,
                       (float)beta1, (float)beta2, (float)eps, bc1, bc2, (float)grad_scale, cc,
                       (step_tensor.has_value() && step_tensor->defined()) ? step_tensor->data_ptr<float>() : nullptr,
                       cur_stream()),
              "ab_adamw");
  g_launches += 1;
}

Tensor grad_sumsq(const Tensor& tensors, const Tensor& chunks) {
  c10::cuda::CUDAGuard guard(tensors.device());
  Tensor out = torch::zeros({1}, tensors.options().dtype(at::kFloat));
  const int nchunks = (int)(chunks.numel() / sizeof(ab::AdamChunk));
  Tensor ws = torch::empty({(int64_t)std::max(1, ab_sumsq_slots(nchunks))}, tensors.options().dtype(at::kFloat));
  AB_CHECK_RC(ab_sumsq(reinterpret_cast<const ab::AdamTensor*>(tensors.data_ptr()),
                       reinterpret_cast<const ab::AdamChunk*>(chunks.data_ptr()), nchunks,
                       out.data_ptr<float>(), ws.data_ptr<float>(), cur_stream()),
              "ab_sumsq");
  g_launches += 2;   // partials + fixed-order reduction
  return out;
}

}  // namespace

// ---- mixture of experts -------------------------------------------------------------------------
static ab::MoePeers moe_peers(const Tensor& local, const std::vector<int64_t>& peer_ptrs, int64_t num_experts) {
  ab::MoePeers p;
  if (peer_ptrs.empty()) {
    p.ptr[0] = local.data_ptr();
    p.experts_per_peer = (int)num_experts;
  } else {
    TORCH_CHECK(peer_ptrs.size() <= ab::kMaxPeersComm && num_experts % (int64_t)peer_ptrs.size() == 0);
    for (size_t i = 0; i < peer_ptrs.size(); ++i) p.ptr[i] = reinterpret_cast<void*>(peer_ptrs[i]);
    p.experts_per_peer = (int)(num_experts / (int64_t)peer_ptrs.size());
  }
  return p;
}

std::vector<Tensor> moe_top2_route(const Tensor& gates, int64_t capacity) {
  TORCH_CHECK(gates.is_cuda() && gates.scalar_type() == at::kFloat && gates.is_contiguous() && gates.dim() == 3);
  c10::cuda::CUDAGuard guard(gates.device());
  const int G = (int)gates.size(0), S = (int)gates.size(1), E = (int)gates.size(2);
  auto opts = gates.options().dtype(at::kLong);
  Tensor expert = torch::empty({G, S, 2}, opts), slot = torch::empty({G, S, 2}, opts);
  AB_CHECK_RC(ab_moe_top2_route(gates.data_ptr<float>(), expert.data_ptr<int64_t>(), slot.data_ptr<int64_t>(), G, S,
                                E, (int)capacity, cur_stream()), "ab_moe_top2_route");
  g_launches += 1;
  return {expert, slot};
}

// d: [E_local, G_total*C, M] (pre-zeroed).  With peer_ptrs: symmetric-memory addresses of d on every peer, the
// global expert count is E_local * peers and this rank's groups start at g_off (fused dispatch + all-to-all).
void moe_dispatch_(const Tensor& x, const Tensor& expert, const Tensor& slot, const OptTensor& weight, Tensor d,
                   int64_t capacity, std::vector<int64_t> peer_ptrs, int64_t g_off) {
  TORCH_CHECK(x.is_contiguous() && expert.is_contiguous() && slot.is_contiguous() && d.is_contiguous());
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && d.scalar_type() == at::kBFloat16 && expert.scalar_type() == at::kLong);
  c10::cuda::CUDAGuard guard(x.device());
  const int G = (int)x.size(0), S = (int)x.size(1), M = (int)x.size(2), K = (int)expert.size(2);
  const int G_total = (int)(d.size(1) / capacity);
  const int64_t E = d.size(0) * (peer_ptrs.empty() ? 1 : (int64_t)peer_ptrs.size());
  ab::MoePeers p = moe_peers(d, peer_ptrs, E);
  AB_CHECK_RC(ab_moe_dispatch(bf16_ptr(x), expert.data_ptr<int64_t>(), slot.data_ptr<int64_t>(), bf16_ptr(weight), &p,
                              G, S, K, M, (int)capacity, (int)g_off, G_total, cur_stream()), "ab_moe_dispatch");
  g_launches += 1;
}

Tensor moe_combine(const Tensor& eo, const Tensor& expert, const Tensor& slot, const OptTensor& weight,
                   std::vector<int64_t> peer_ptrs, int64_t g_off) {
  TORCH_CHECK(eo.is_contiguous() && expert.is_contiguous() && slot.is_contiguous());
  TORCH_CHECK(eo.scalar_type() == at::kBFloat16 && expert.scalar_type() == at::kLong);
  c10::cuda::CUDAGuard guard(eo.device());
  const int G = (int)expert.size(0), S = (int)expert.size(1), K = (int)expert.size(2), M = (int)eo.size(2);
  const int64_t peers = peer_ptrs.empty() ? 1 : (int64_t)peer_ptrs.size();
  const int G_total = peer_ptrs.empty() ? G : G * (int)peers;
  const int C = (int)(eo.size(1) / G_total);
  ab::MoePeers p = moe_peers(eo, peer_ptrs, eo.size(0) * peers);
  Tensor out = torch::empty({G, S, M}, eo.options());
  AB_CHECK_RC(ab_moe_combine(&p, expert.data_ptr<int64_t>(), slot.data_ptr<int64_t>(), bf16_ptr(weight),
                             reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), G, S, K, M, C, (int)g_off, G_total,
                             cur_stream()), "ab_moe_combine");
  g_launches += 1;
  return out;
}

Tensor moe_combine_wgrad(const Tensor& dout, const Tensor& eo, const Tensor& expert, const Tensor& slot,
                         std::vector<int64_t> peer_ptrs, int64_t g_off) {
  TORCH_CHECK(eo.is_contiguous() && expert.is_contiguous() && slot.is_contiguous() && dout.is_contiguous());
  TORCH_CHECK(eo.scalar_type() == at::kBFloat16 && dout.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(eo.device());
  const int G = (int)expert.size(0), S = (int)expert.size(1), K = (int)expert.size(2), M = (int)eo.size(2);
  const int64_t peers = peer_ptrs.empty() ? 1 : (int64_t)peer_ptrs.size();
  const int G_total = peer_ptrs.empty() ? G : G * (int)peers;
  const int C = (int)(eo.size(1) / G_total);
  ab::MoePeers p = moe_peers(eo, peer_ptrs, eo.size(0) * peers);
  Tensor dw = torch::empty({G, S, K}, dout.options());
  AB_CHECK_RC(ab_moe_combine_wgrad(bf16_ptr(dout), &p, expert.data_ptr<int64_t>(), slot.data_ptr<int64_t>(),
                                   reinterpret_cast<__nv_bfloat16*>(dw.data_ptr()), G, S, K, M, C, (int)g_off,
                                   G_total, cur_stream()), "ab_moe_combine_wgrad");
  g_launches += 1;
  return dw;
}

// ---- fp8 serving GEMM ---------------------------------------------------------------------------
// The row quantisers read x 16 bytes at a time (ld_nc_v4): every row must start on a 16-byte boundary.
void check_rows_16b(const Tensor& x, const char* what) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.stride(1) == 1, what,
              ": x must be a 2-D CUDA bf16 tensor with a contiguous inner dim");
  TORCH_CHECK(x.stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, what,
              ": x needs a row stride that is a multiple of 8 and a 16-byte aligned base");
}

// Per-row e4m3 quantisation of the activations: x bf16 [M, K] -> (q e4m3 [M, K], sx fp32 [M]), x ~ q * sx[m]
std::vector<Tensor> quantize_e4m3(const Tensor& x) {
  check_rows_16b(x, "quantize_e4m3");
  c10::cuda::CUDAGuard guard(x.device());
  const int M = (int)x.size(0), K = (int)x.size(1);
  TORCH_CHECK(K % 16 == 0, "quantize_e4m3: K must be a multiple of 16");
  Tensor q = torch::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor sx = torch::empty({M}, x.options().dtype(at::kFloat));
  AB_CHECK_RC(ab_quantize_rows_e4m3(bf16_ptr(x), reinterpret_cast<uint8_t*>(q.data_ptr()), sx.data_ptr<float>(), M, K,
                                    x.stride(0), cur_stream()), "ab_quantize_rows_e4m3");
  g_launches += 1;
  return {q, sx};
}

// y = act((xq . wq^T) * sx[m] * sw[n] + bias): xq e4m3 [M, K], sx fp32 [M], wq e4m3 [N, K], sw fp32 [N]
Tensor gemm_fp8_q(const Tensor& xq, const Tensor& sx, const Tensor& wq, const Tensor& sw, const OptTensor& bias,
                  int64_t act) {
  TORCH_CHECK(xq.is_cuda() && xq.scalar_type() == at::kFloat8_e4m3fn && xq.dim() == 2 && xq.is_contiguous(), "gemm_fp8: xq");
  TORCH_CHECK(wq.is_cuda() && wq.scalar_type() == at::kFloat8_e4m3fn && wq.dim() == 2 && wq.is_contiguous(),
              "gemm_fp8: w must be contiguous e4m3");
  const int M = (int)xq.size(0), K = (int)xq.size(1), N = (int)wq.size(0);
  TORCH_CHECK(wq.size(1) == K && K % 16 == 0 && N % 8 == 0, "gemm_fp8: shapes");
  TORCH_CHECK(sx.scalar_type() == at::kFloat && sx.is_contiguous() && sx.numel() == M, "gemm_fp8: sx must be fp32 [M]");
  TORCH_CHECK(sw.scalar_type() == at::kFloat && sw.is_contiguous() && sw.numel() == N, "gemm_fp8: w_scale must be fp32 [N]");
  if (bias.has_value() && bias->defined())
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() && bias->numel() == N &&
                    reinterpret_cast<uintptr_t>(bias->data_ptr()) % 4 == 0,
                "gemm_fp8: bias must be a contiguous, 4-byte aligned bf16 [N]");
  c10::cuda::CUDAGuard guard(xq.device());
  Tensor out = torch::empty({M, N}, xq.options().dtype(at::kBFloat16));
  AB_CHECK_RC(ab_gemm_fp8(reinterpret_cast<const uint8_t*>(xq.data_ptr()), reinterpret_cast<const uint8_t*>(wq.data_ptr()),
                          sx.data_ptr<float>(), sw.data_ptr<float>(), bf16_ptr(bias),
                          reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), M, N, K, N, (int)act, cur_stream()),
              "ab_gemm_fp8");
  g_launches += 1;
  return out;
}

// y = act((quantize_e4m3(x) . w_fp8^T) * sx * sw + bias): x bf16 [M, K], w e4m3 [N, K], w_scale fp32 [N]
Tensor gemm_fp8(const Tensor& x, const Tensor& w, const Tensor& w_scale, const OptTensor& bias, int64_t act) {
  check_rows_16b(x, "gemm_fp8");
  TORCH_CHECK(w.dim() == 2 && w.size(1) == x.size(1), "gemm_fp8: shapes");
  if (bias.has_value() && bias->defined())   // checked before the quantiser launches
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->numel() == w.size(0), "gemm_fp8: bias must be bf16 [N]");
  auto qs = quantize_e4m3(x);
  return gemm_fp8_q(qs[0], qs[1], w, w_scale, bias, act);
}

// Cross-mesh resharding pack / unpack (pack_sm90.cu): `views` are <= 4-D slices with a contiguous innermost dim; tile k
// lives in `flat` (uint8) at the 16-byte aligned running offset.  unpack = false: views -> flat; true: flat -> views.
void pack_tiles(const std::vector<Tensor>& views, Tensor flat, bool unpack) {
  TORCH_CHECK(flat.is_cuda() && flat.scalar_type() == at::kByte && flat.is_contiguous(), "pack_tiles: flat must be uint8");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(flat.data_ptr()) % 16 == 0, "pack_tiles: flat must be 16-byte aligned");
  c10::cuda::CUDAGuard guard(flat.device());
  char* base = reinterpret_cast<char*>(flat.data_ptr());
  int64_t off = 0;
  size_t k = 0;
  while (k < views.size()) {
    ab::PackArgs a;
    a.num_tiles = 0;
    for (; k < views.size() && a.num_tiles < ab::kMaxPackTiles; ++k) {
      const Tensor& v = views[k];
      TORCH_CHECK(v.is_cuda() && v.dim() >= 1 && v.dim() <= 4 && v.stride(-1) == 1 && v.numel() > 0,
                  "pack_tiles: views must be non-empty <= 4-D CUDA slices with a contiguous innermost dim");
      const int64_t es = v.element_size();
      ab::PackTile& t = a.tiles[a.num_tiles++];
      const int pad = 4 - (int)v.dim();
      for (int d = 0; d < 4; ++d) t.shape[d] = d < pad ? 1 : v.size(d - pad);
      for (int d = 0; d < 3; ++d) t.stride[d] = d < pad ? 0 : v.stride(d - pad) * es;
      t.shape[3] *= es;
      t.strided = reinterpret_cast<char*>(v.data_ptr());
      t.packed = base + off;
      const int64_t bytes = v.numel() * es;
      TORCH_CHECK(off + bytes <= flat.numel(), "pack_tiles: flat buffer too small");
      bool vec = t.shape[3] % 16 == 0 && reinterpret_cast<uintptr_t>(t.strided) % 16 == 0;
      for (int d = 0; d < 3; ++d) vec = vec && (t.stride[d] % 16 == 0);
      t.vec16 = vec ? 1 : 0;
      off += (bytes + 15) / 16 * 16;
    }
    AB_CHECK_RC(ab_pack_tiles(&a, unpack ? 1 : 0, cur_stream()), "ab_pack_tiles");
    g_launches += 1;
  }
}

// Block-scaled MXFP8: e4m3 elements + one UE8M0 scale per 32 K elements, scale atoms of 128 rows x 4 K-blocks
// (gemm_sm90.cu).  Returns (q [M, K] e4m3, sf uint8 [ceil(M/128), ceil(K/128), 512]).
std::vector<Tensor> quantize_mxfp8(const Tensor& x) {
  check_rows_16b(x, "quantize_mxfp8");
  c10::cuda::CUDAGuard guard(x.device());
  const int M = (int)x.size(0), K = (int)x.size(1);
  TORCH_CHECK(K % 32 == 0, "quantize_mxfp8: K must be a multiple of 32");
  Tensor q = torch::empty({M, K}, x.options().dtype(at::kFloat8_e4m3fn));
  Tensor sf = torch::full({(M + 127) / 128, (K + 127) / 128, 512}, 127, x.options().dtype(at::kByte));
  AB_CHECK_RC(ab_quantize_rows_mxfp8(bf16_ptr(x), reinterpret_cast<uint8_t*>(q.data_ptr()), sf.data_ptr<uint8_t>(), M, K,
                                     x.stride(0), cur_stream()), "ab_quantize_rows_mxfp8");
  g_launches += 1;
  return {q, sf};
}

Tensor gemm_mxfp8_q(const Tensor& xq, const Tensor& x_sf, const Tensor& wq, const Tensor& w_sf, const OptTensor& bias,
                    int64_t act) {
  TORCH_CHECK(xq.is_cuda() && xq.scalar_type() == at::kFloat8_e4m3fn && xq.dim() == 2 && xq.is_contiguous(), "gemm_mxfp8: xq");
  TORCH_CHECK(wq.is_cuda() && wq.scalar_type() == at::kFloat8_e4m3fn && wq.dim() == 2 && wq.is_contiguous(), "gemm_mxfp8: wq");
  const int M = (int)xq.size(0), K = (int)xq.size(1), N = (int)wq.size(0);
  TORCH_CHECK(wq.size(1) == K && K % 32 == 0 && N % 8 == 0, "gemm_mxfp8: shapes");
  const int64_t ka = (K + 127) / 128;
  TORCH_CHECK(x_sf.scalar_type() == at::kByte && x_sf.is_contiguous() && x_sf.numel() == (int64_t)((M + 127) / 128) * ka * 512,
              "gemm_mxfp8: x scale atoms");
  TORCH_CHECK(w_sf.scalar_type() == at::kByte && w_sf.is_contiguous() && w_sf.numel() == (int64_t)((N + 127) / 128) * ka * 512,
              "gemm_mxfp8: w scale atoms");
  if (bias.has_value() && bias->defined())
    TORCH_CHECK(bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() && bias->numel() == N, "gemm_mxfp8: bias");
  c10::cuda::CUDAGuard guard(xq.device());
  Tensor out = torch::empty({M, N}, xq.options().dtype(at::kBFloat16));
  AB_CHECK_RC(ab_gemm_mxfp8(reinterpret_cast<const uint8_t*>(xq.data_ptr()), x_sf.data_ptr<uint8_t>(),
                            reinterpret_cast<const uint8_t*>(wq.data_ptr()), w_sf.data_ptr<uint8_t>(), bf16_ptr(bias),
                            reinterpret_cast<__nv_bfloat16*>(out.data_ptr()), M, N, K, N, (int)act, cur_stream()),
              "ab_gemm_mxfp8");
  g_launches += 1;
  return out;
}

// y = act(x . dequant(wq, w_sf)^T + b): activations are block-quantised on the fly
Tensor gemm_mxfp8(const Tensor& x, const Tensor& wq, const Tensor& w_sf, const OptTensor& bias, int64_t act) {
  auto qs = quantize_mxfp8(x);
  return gemm_mxfp8_q(qs[0], qs[1], wq, w_sf, bias, act);
}

// Decode-step GEMV: x [M<=8, K] bf16, w [N, K] e4m3 (with w_scale [N]) or bf16.
Tensor gemv_decode(const Tensor& x, const Tensor& w, const OptTensor& w_scale, const OptTensor& bias,
                   const OptTensor& residual, int64_t act, const OptTensor& ln_gamma, const OptTensor& ln_beta,
                   double ln_eps) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.scalar_type() == at::kBFloat16 && x.stride(1) == 1 &&
                  reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "gemv_decode: x (16-byte aligned rows)");
  const bool fp8 = w.scalar_type() == at::kFloat8_e4m3fn;
  TORCH_CHECK((fp8 || w.scalar_type() == at::kBFloat16) && w.dim() == 2 && w.is_contiguous() && w.size(1) == x.size(1),
              "gemv_decode: w must be contiguous [N, K] e4m3 / bf16");
  c10::cuda::CUDAGuard guard(x.device());
  ab::GemvArgs a;
  a.M = (int)x.size(0); a.K = (int)x.size(1); a.N = (int)w.size(0);
  a.x = bf16_ptr(x); a.w = w.data_ptr(); a.fp8 = fp8 ? 1 : 0; a.act = (int)act;
  a.ldx = x.stride(0);
  if (fp8) {
    TORCH_CHECK(w_scale.has_value() && w_scale->defined() && w_scale->scalar_type() == at::kFloat &&
                w_scale->numel() == a.N && w_scale->is_contiguous(), "gemv_decode: w_scale");
    a.w_scale = w_scale->data_ptr<float>();
  }
  a.bias = bf16_ptr(bias);
  Tensor y = torch::empty({a.M, a.N}, x.options());
  a.y = reinterpret_cast<__nv_bfloat16*>(y.data_ptr());
  a.ldy = a.N;
  if (residual.has_value() && residual->defined()) {
    TORCH_CHECK(residual->dim() == 2 && residual->size(0) == a.M && residual->size(1) == a.N && residual->stride(1) == 1 &&
                residual->scalar_type() == at::kBFloat16, "gemv_decode: residual");
    a.residual = bf16_ptr(residual);
    a.ldr = residual->stride(0);
  }
  if (ln_gamma.has_value() && ln_gamma->defined()) {
    TORCH_CHECK(ln_beta.has_value() && ln_beta->defined() && ln_gamma->scalar_type() == at::kBFloat16 &&
                ln_beta->scalar_type() == at::kBFloat16 && ln_gamma->is_contiguous() && ln_beta->is_contiguous() &&
                ln_gamma->numel() == a.K && ln_beta->numel() == a.K, "gemv_decode: layer-norm gamma / beta must be bf16 [K]");
    a.ln_gamma = bf16_ptr(ln_gamma);
    a.ln_beta = bf16_ptr(ln_beta);
    a.ln_eps = (float)ln_eps;
  }
  AB_CHECK_RC(ab_gemv_decode(&a, cur_stream()), "ab_gemv_decode");
  g_launches += 1;
  return y;
}

// Decode-step attention, cache append fused: q / k_new / v_new [B, 1, heads, D] views, caches [B, S_max, heads, D].
Tensor decode_attention(const Tensor& q, const Tensor& k_new, const Tensor& v_new, Tensor k_cache, Tensor v_cache,
                        const Tensor& kv_len, double scale) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 4 && q.size(1) == 1 && q.scalar_type() == at::kBFloat16 && q.stride(3) == 1,
              "decode_attention: q must be bf16 [B, 1, heads, D]");
  TORCH_CHECK(k_new.sizes() == q.sizes() && v_new.sizes() == q.sizes() && k_new.scalar_type() == at::kBFloat16 &&
              v_new.scalar_type() == at::kBFloat16 && k_new.stride(3) == 1 && v_new.stride(3) == 1 &&
              k_new.stride(0) == v_new.stride(0) && k_new.stride(2) == v_new.stride(2),
              "decode_attention: k_new / v_new must be bf16 [B, 1, heads, D] with equal strides");
  TORCH_CHECK(k_cache.dim() == 4 && k_cache.scalar_type() == at::kBFloat16 && v_cache.scalar_type() == at::kBFloat16 &&
              k_cache.sizes() == v_cache.sizes() && k_cache.strides() == v_cache.strides() && k_cache.size(0) == q.size(0) &&
              k_cache.size(2) == q.size(2) && k_cache.size(3) == q.size(3) && k_cache.stride(3) == 1 &&
              k_cache.stride(2) == k_cache.size(3), "decode_attention: caches must be bf16 [B, S_max, heads, D], rows dense");
  TORCH_CHECK(kv_len.is_cuda() && kv_len.scalar_type() == at::kInt && kv_len.numel() == 1,
              "decode_attention: kv_len must be an int32 CUDA scalar");
  c10::cuda::CUDAGuard guard(q.device());
  ab::DecodeAttnArgs a;
  a.q = bf16_ptr(q); a.k_new = bf16_ptr(k_new); a.v_new = bf16_ptr(v_new);
  a.k_cache = reinterpret_cast<__nv_bfloat16*>(k_cache.data_ptr());
  a.v_cache = reinterpret_cast<__nv_bfloat16*>(v_cache.data_ptr());
  a.kv_len = kv_len.data_ptr<int>();
  a.B = (int)q.size(0); a.heads = (int)q.size(2); a.D = (int)q.size(3); a.S_max = (int)k_cache.size(1);
  a.q_stride_b = q.stride(0); a.q_stride_h = q.stride(2);
  a.new_stride_b = k_new.stride(0); a.new_stride_h = k_new.stride(2);
  a.cache_stride_b = k_cache.stride(0); a.cache_stride_s = k_cache.stride(1);
  a.scale = (float)scale;
  Tensor o = torch::empty({a.B, 1, a.heads, a.D}, q.options());
  a.o = reinterpret_cast<__nv_bfloat16*>(o.data_ptr());
  // split the key range so that ~2 CTAs per SM stream the cache (the length is only known on the device)
  const int bh = a.B * a.heads;
  a.splits = std::max(1, std::min(16, (2 * ab::num_sms() + bh - 1) / bh));
  Tensor ws;
  if (a.splits > 1) {
    // arrival counters: one persistent zeroed buffer per device; the merging CTA resets its counter
    static std::unordered_map<int, Tensor> counters;
    const int dev = q.get_device();
    auto it = counters.find(dev);
    if (it == counters.end() || it->second.numel() < bh)
      it = counters.insert_or_assign(dev, torch::zeros({std::max(bh, 4096)}, q.options().dtype(at::kInt))).first;
    a.counters = it->second.data_ptr<int>();
    ws = torch::empty({(int64_t)bh * a.splits * (a.D + 2)}, q.options().dtype(at::kFloat));
    a.ws = ws.data_ptr<float>();
  }
  AB_CHECK_RC(ab_decode_attention(&a, cur_stream()), "ab_decode_attention");
  g_launches += 1;
  return o;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "alpa_b200 sm_90a kernels";
  m.def("launch_count", []() { return (long long)g_launches.load(); });
  // kernels replayed from a captured CUDA graph are launched by the driver, not through these bindings: the executor
  // adds the number it recorded at capture time for every replay
  m.def("add_launches", [](long long n) { g_launches += n; });
  m.def("gemm", &gemm, py::arg("a"), py::arg("b"), py::arg("trans_a") = false,
        py::arg("trans_b") = false, py::arg("out") = py::none(), py::arg("bias") = py::none(),
        py::arg("residual") = py::none(), py::arg("aux_out") = py::none(),
        py::arg("aux_in") = py::none(), py::arg("act") = 0, py::arg("alpha") = 1.0,
        py::arg("accumulate") = false, py::arg("out_fp32") = false, py::arg("block_n") = 0,
        py::arg("epilogue") = "auto");
  m.def("gemm_scatter", &gemm_scatter, py::arg("a"), py::arg("b"), py::arg("trans_b"), py::arg("peer_ptrs"),
        py::arg("flag_ptrs"), py::arg("slot"), py::arg("rows_per_dst"), py::arg("ldc"), py::arg("m_block_rotate"),
        py::arg("max_ctas"), py::arg("trans_a") = false);
  m.def("rs_reduce", &rs_reduce);
  m.def("ag_push", &ag_push);
  m.def("gemm_wait_a", &gemm_wait_a);
  m.def("allreduce_multimem", &allreduce_multimem, py::arg("mc_ptr"), py::arg("numel"), py::arg("rank"), py::arg("tp"),
        py::arg("ctas") = 0);
  m.def("peer_barrier", &peer_barrier);
  m.def("peer_barrier_auto", &peer_barrier_auto);
  m.def("allreduce_oneshot", &allreduce_oneshot, py::arg("x"), py::arg("sym_local_ptr"), py::arg("mc_ptr"),
        py::arg("half_stride"), py::arg("out"), py::arg("flag_ptrs"), py::arg("counter"), py::arg("rank"),
        py::arg("residual") = py::none());
  m.def("attention_fwd", &attention_fwd, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("scale"), py::arg("causal"),
        py::arg("kv_len") = py::none());
  m.def("attention_bwd", &attention_bwd, py::arg("d_o"), py::arg("q"), py::arg("k"), py::arg("v"), py::arg("o"),
        py::arg("lse"), py::arg("scale"), py::arg("causal"), py::arg("dq_out") = py::none(),
        py::arg("dk_out") = py::none(), py::arg("dv_out") = py::none());
  m.def("layernorm_fwd", &layernorm_fwd);
  m.def("layernorm_bwd", &layernorm_bwd);
  m.def("ce_stats", &ce_stats);
  m.def("ce_grad_", &ce_grad_);
  m.def("ragged_attention", &ragged_attention, py::arg("q"), py::arg("k_cache"), py::arg("v_cache"), py::arg("seq_start"),
        py::arg("ctx_len"), py::arg("scale"), py::arg("max_ctx"), py::arg("alibi") = py::none());
  m.def("dropout", &dropout);
  m.def("embedding_fwd", &embedding_fwd);
  m.def("embedding_bwd_", &embedding_bwd_);
  m.def("colsum_", &colsum_);
  m.def("adam_build_tables", &adam_build_tables);
  m.def("adamw_step", &adamw_step, py::arg("tensors"), py::arg("chunks"), py::arg("lr"), py::arg("beta1"),
        py::arg("beta2"), py::arg("eps"), py::arg("step"), py::arg("grad_scale"),
        py::arg("clip_coef") = py::none(), py::arg("step_tensor") = py::none());
  m.def("grad_sumsq", &grad_sumsq);
  m.def("quantize_e4m3", &quantize_e4m3);
  m.def("gemm_fp8_q", &gemm_fp8_q);
  m.def("gemm_fp8", &gemm_fp8);
  m.def("pack_tiles", &pack_tiles, py::arg("views"), py::arg("flat"), py::arg("unpack") = false);
  m.def("quantize_mxfp8", &quantize_mxfp8);
  m.def("gemm_mxfp8", &gemm_mxfp8);
  m.def("gemm_mxfp8_q", &gemm_mxfp8_q);
  m.def("gemv_decode", &gemv_decode, py::arg("x"), py::arg("w"), py::arg("w_scale") = py::none(),
        py::arg("bias") = py::none(), py::arg("residual") = py::none(), py::arg("act") = 0,
        py::arg("ln_gamma") = py::none(), py::arg("ln_beta") = py::none(), py::arg("ln_eps") = 1e-5);
  m.def("decode_attention", &decode_attention);
  m.def("moe_top2_route", &moe_top2_route);
  m.def("moe_dispatch_", &moe_dispatch_, py::arg("x"), py::arg("expert"), py::arg("slot"), py::arg("weight"),
        py::arg("d"), py::arg("capacity"), py::arg("peer_ptrs") = std::vector<int64_t>(), py::arg("g_off") = 0);
  m.def("moe_combine", &moe_combine, py::arg("eo"), py::arg("expert"), py::arg("slot"), py::arg("weight"),
        py::arg("peer_ptrs") = std::vector<int64_t>(), py::arg("g_off") = 0);
  m.def("moe_combine_wgrad", &moe_combine_wgrad, py::arg("dout"), py::arg("eo"), py::arg("expert"), py::arg("slot"),
        py::arg("peer_ptrs") = std::vector<int64_t>(), py::arg("g_off") = 0);
}
