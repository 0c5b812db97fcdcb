"""GPT language model built from the alpa_b200 primitives.

Architecture parity with the reference's benchmark model (alpa/model/gpt_model.py:19-93 on top of
alpa/model/bert_model.py: word+position embeddings -> LayerNorm -> L x [self-attention, dense,
residual+LayerNorm, dense+GELU, dense, residual+LayerNorm] (post-LN) -> vocabulary projection + bias).
The reference attends bidirectionally with an all-ones mask in its GPT benchmark
(benchmark_one_case_gpt_bert.py:142-148); `causal=True` gives the usual decoder masking.

H100 mapping: fused QKV projection (features ordered (head, {q,k,v}, D) so tensor-parallel splits are
head splits; with grouped-query attention (K/V head, {G query heads, k, v}, D)), packed flash attention, GELU / bias / pre-activation fused into GEMM epilogues,
residual-add fused into LayerNorm, per-token fused cross-entropy.

`arch="llama"` builds the Llama-style decoder instead: no position table, pre-RMSNorm blocks with bias-free linears,
rotary position embeddings on the packed QKV tensor, a SwiGLU MLP whose fc1 output holds (gate, up) in interleaved
pairs, and the residual adds fused into the next RMSNorm (`add_rms_norm`).  `llama_config_from_hf` /
`llama_params_from_hf` load Hugging Face Llama checkpoints into it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from alpa_b200 import ops
from alpa_b200.parallel.pipeline.primitive_def import mark_pipeline_boundary


@dataclass
class GPTConfig:
    vocab_size: int = 51200
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    # grouped-query attention: K/V heads shared by groups of num_attention_heads // num_key_value_heads query heads
    # (None or num_attention_heads: multi-head attention)
    num_key_value_heads: Optional[int] = None
    intermediate_size: Optional[int] = None
    max_position_embeddings: int = 1024
    layer_norm_eps: float = 1e-12
    initializer_range: float = 0.02
    # None: the architecture's own masking -- bidirectional for "gpt" (reference benchmark: all-ones mask), causal for
    # "llama"
    causal: Optional[bool] = None
    tie_word_embeddings: bool = False
    add_manual_pipeline_markers: bool = False  # mark a layer boundary every `pipeline_mp_size` blocks
    pipeline_mp_size: int = 0
    gradient_checkpointing: bool = False
    hidden_dropout_prob: float = 0.0           # counter-based dropout (ops.dropout) after proj / fc2 when a seed is passed
    dtype: torch.dtype = torch.bfloat16
    # "gpt": the reference's post-LN GPT block; "llama": pre-RMSNorm, rotary embeddings, SwiGLU, no biases
    # (layer_norm_eps is the RMSNorm eps, max_position_embeddings is unused)
    arch: str = "gpt"
    rope_theta: float = 10000.0

    def __post_init__(self):
        if self.intermediate_size is None:
            self.intermediate_size = 4 * self.hidden_size
        if self.arch not in ("gpt", "llama"):
            raise ValueError(f"arch must be 'gpt' or 'llama', not {self.arch!r}")
        if self.causal is None:
            self.causal = self.arch == "llama"
        if self.arch == "llama" and self.hidden_dropout_prob > 0.0:
            raise ValueError("arch='llama' has no hidden dropout")
        assert self.hidden_size % self.num_attention_heads == 0
        kv = self.num_key_value_heads
        assert kv is None or (kv > 0 and self.num_attention_heads % kv == 0), \
            "num_key_value_heads must divide num_attention_heads"

    @property
    def qkv_features(self) -> int:
        """Output features of the fused QKV projection: (G + 2) Hkv D, which is 3 H for multi-head attention."""
        kv = self.num_key_value_heads or self.num_attention_heads
        return (self.num_attention_heads + 2 * kv) * (self.hidden_size // self.num_attention_heads)


# (S, H, L, heads, V) of the reference's benchmark suite (benchmark/alpa/suite_manual_gpt.py:16-27)
GPT_SPECS = {
    "test-tiny": (32, 64, 4, 4, 512),          # CPU smoke tests of the benchmark / planning paths
    "125M": (1024, 768, 12, 12, 51200),
    "350M": (1024, 1024, 24, 16, 51200),
    "760M": (1024, 1536, 24, 16, 51200),
    "1.3B": (1024, 2048, 24, 32, 51200),
    "2.6B": (1024, 2560, 32, 32, 51200),
    "6.7B": (1024, 4096, 32, 32, 51200),
    "15B": (1024, 5120, 48, 40, 51200),
    "39B": (1024, 8192, 48, 64, 51200),
    "76B": (1024, 10240, 60, 80, 51200),
}


def config_from_spec(name: str, **kw) -> GPTConfig:
    s, h, l, heads, v = GPT_SPECS[name]
    return GPTConfig(vocab_size=v, hidden_size=h, num_hidden_layers=l, num_attention_heads=heads,
                     max_position_embeddings=s, **kw)


class GPTBlock(nn.Module):
    def __init__(self, cfg: GPTConfig, device=None):
        super().__init__()
        H, I = cfg.hidden_size, cfg.intermediate_size
        kw = dict(device=device, dtype=cfg.dtype)
        std = cfg.initializer_range
        self.cfg = cfg
        self.qkv_w = nn.Parameter(torch.randn(cfg.qkv_features, H, **kw) * std)
        self.qkv_b = nn.Parameter(torch.zeros(cfg.qkv_features, **kw))
        self.proj_w = nn.Parameter(torch.randn(H, H, **kw) * std)
        self.proj_b = nn.Parameter(torch.zeros(H, **kw))
        self.ln1_g = nn.Parameter(torch.ones(H, **kw))
        self.ln1_b = nn.Parameter(torch.zeros(H, **kw))
        self.fc1_w = nn.Parameter(torch.randn(I, H, **kw) * std)
        self.fc1_b = nn.Parameter(torch.zeros(I, **kw))
        self.fc2_w = nn.Parameter(torch.randn(H, I, **kw) * std)
        self.fc2_b = nn.Parameter(torch.zeros(H, **kw))
        self.ln2_g = nn.Parameter(torch.ones(H, **kw))
        self.ln2_b = nn.Parameter(torch.zeros(H, **kw))

    def forward(self, x, dropout_seed=None, layer_idx: int = 0):
        cfg = self.cfg
        B, S, H = x.shape
        nh = cfg.num_attention_heads
        D = H // nh
        drop = dropout_seed is not None and getattr(cfg, "hidden_dropout_prob", 0.0) > 0.0
        # features ordered (K/V head, {its G query heads, k, v}, D): a column split is a split over K/V heads
        kv = cfg.num_key_value_heads or nh
        qkv = ops.linear(x, self.qkv_w, self.qkv_b).view(B, S, kv, nh // kv + 2, D)
        o, _ = ops.attention_gqa_packed(qkv, 1.0 / math.sqrt(D), cfg.causal)
        a = ops.linear(o.view(B, S, H), self.proj_w, self.proj_b)
        if drop:
            a = ops.dropout_like(a, cfg.hidden_dropout_prob, dropout_seed, stream=2 * layer_idx + 1)
        x1, _, _, _ = ops.add_layer_norm(a, x, self.ln1_g, self.ln1_b, cfg.layer_norm_eps)
        h, _ = ops.linear_act(x1, self.fc1_w, self.fc1_b, "gelu")
        m = ops.linear(h, self.fc2_w, self.fc2_b)
        if drop:
            m = ops.dropout_like(m, cfg.hidden_dropout_prob, dropout_seed, stream=2 * layer_idx + 2)
        x2, _, _, _ = ops.add_layer_norm(m, x1, self.ln2_g, self.ln2_b, cfg.layer_norm_eps)
        return x2


class LlamaBlock(nn.Module):
    """Pre-RMSNorm block: x + attn(rope(rms(x))), then + swiglu_mlp(rms(.)).  The residual stream arrives as
    (branch output, residual), or (x, None) for the first block, and leaves the same way, so that every residual add is
    fused into the RMSNorm that follows it."""

    def __init__(self, cfg: GPTConfig, device=None):
        super().__init__()
        H, I = cfg.hidden_size, cfg.intermediate_size
        kw = dict(device=device, dtype=cfg.dtype)
        std = cfg.initializer_range
        self.cfg = cfg
        self.ln1_g = nn.Parameter(torch.ones(H, **kw))
        self.qkv_w = nn.Parameter(torch.randn(cfg.qkv_features, H, **kw) * std)
        self.proj_w = nn.Parameter(torch.randn(H, H, **kw) * std)
        self.ln2_g = nn.Parameter(torch.ones(H, **kw))
        self.fc1_w = nn.Parameter(torch.randn(2 * I, H, **kw) * std)   # rows (2j, 2j + 1) = (gate j, up j)
        self.fc2_w = nn.Parameter(torch.randn(H, I, **kw) * std)

    def forward(self, a, r, position_ids):
        cfg = self.cfg
        B, S, H = a.shape
        nh = cfg.num_attention_heads
        kv, D = cfg.num_key_value_heads or nh, H // nh
        if r is None:
            h, _ = ops.rms_norm(a, self.ln1_g, cfg.layer_norm_eps)
            x = a
        else:
            h, x, _ = ops.add_rms_norm(a, r, self.ln1_g, cfg.layer_norm_eps)
        qkv = ops.linear(h, self.qkv_w).view(B, S, kv, nh // kv + 2, D)
        qkv = ops.rotary_packed(qkv, position_ids, cfg.rope_theta, False)
        o, _ = ops.attention_gqa_packed(qkv, 1.0 / math.sqrt(D), cfg.causal)
        attn = ops.linear(o.view(B, S, H), self.proj_w)
        h2, x2, _ = ops.add_rms_norm(attn, x, self.ln2_g, cfg.layer_norm_eps)
        gu = ops.linear(h2, self.fc1_w).view(B, S, cfg.intermediate_size, 2)
        return ops.linear(ops.swiglu(gu), self.fc2_w), x2


class GPTModel(nn.Module):
    """`forward(input_ids, position_ids) -> logits [B, S, V]`."""

    def __init__(self, cfg: GPTConfig, device=None):
        super().__init__()
        self.cfg = cfg
        kw = dict(device=device, dtype=cfg.dtype)
        std = cfg.initializer_range
        H = cfg.hidden_size
        llama = cfg.arch == "llama"
        self.wte = nn.Parameter(torch.randn(cfg.vocab_size, H, **kw) * std)
        if not llama:
            self.wpe = nn.Parameter(torch.randn(cfg.max_position_embeddings, H, **kw) * std)
            self.emb_ln_g = nn.Parameter(torch.ones(H, **kw))
            self.emb_ln_b = nn.Parameter(torch.zeros(H, **kw))
        block = LlamaBlock if llama else GPTBlock
        self.blocks = nn.ModuleList([block(cfg, device) for _ in range(cfg.num_hidden_layers)])
        if llama:
            self.ln_f_g = nn.Parameter(torch.ones(H, **kw))
        if not cfg.tie_word_embeddings:
            self.decoder_w = nn.Parameter(torch.randn(cfg.vocab_size, H, **kw) * std)
        if not llama:
            self.decoder_b = nn.Parameter(torch.zeros(cfg.vocab_size, **kw))

    def _boundary(self, i: int) -> bool:
        """Whether a manual pipeline boundary precedes block i."""
        cfg = self.cfg
        if not (cfg.add_manual_pipeline_markers and cfg.pipeline_mp_size > 1 and i > 0):
            return False
        per = max(1, cfg.num_hidden_layers // cfg.pipeline_mp_size)
        return i % per == 0 and i // per < cfg.pipeline_mp_size

    def _llama_hidden_states(self, input_ids, position_ids):
        a, r = ops.embedding(input_ids, self.wte), None
        for i, blk in enumerate(self.blocks):
            if self._boundary(i):
                a, r = mark_pipeline_boundary(a, r)
            a, r = blk(a, r, position_ids)
        if r is None:
            return ops.rms_norm(a, self.ln_f_g, self.cfg.layer_norm_eps)[0]
        return ops.add_rms_norm(a, r, self.ln_f_g, self.cfg.layer_norm_eps)[0]

    def hidden_states(self, input_ids, position_ids, dropout_seed=None):
        cfg = self.cfg
        if cfg.arch == "llama":
            return self._llama_hidden_states(input_ids, position_ids)
        x = ops.embedding(input_ids, self.wte) + ops.embedding(position_ids, self.wpe)
        x, _, _ = ops.layer_norm(x, self.emb_ln_g, self.emb_ln_b, cfg.layer_norm_eps)
        if dropout_seed is not None and cfg.hidden_dropout_prob > 0.0:
            x = ops.dropout_like(x, cfg.hidden_dropout_prob, dropout_seed, stream=0)
        for i, blk in enumerate(self.blocks):
            if self._boundary(i):
                x = mark_pipeline_boundary(x)
            x = blk(x, dropout_seed, i) if dropout_seed is not None else blk(x)
        return x

    def forward(self, input_ids, position_ids, dropout_seed=None):
        """`dropout_seed`: int64 scalar tensor (e.g. from the step counter) enables hidden-state dropout in training."""
        x = self.hidden_states(input_ids, position_ids, dropout_seed)
        w = self.wte if self.cfg.tie_word_embeddings else self.decoder_w
        return ops.linear(x, w, getattr(self, "decoder_b", None))


def gpt_lm_loss(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """Masked mean token cross-entropy (reference loss: benchmark_one_case_gpt_bert.py:106-110:
    positions with label <= 0 are ignored)."""
    V = logits.shape[-1]
    loss, _ = ops.cross_entropy(logits.reshape(-1, V), labels.reshape(-1))
    mask = (labels.reshape(-1) > 0).to(loss.dtype)
    return (loss * mask).sum() / mask.sum().clamp(min=1.0)


def num_params(cfg: GPTConfig) -> int:
    H, I, V, L = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.num_hidden_layers
    F = cfg.qkv_features
    if cfg.arch == "llama":
        per_layer = H + F * H + H * H + H + 2 * I * H + I * H
        return L * per_layer + V * H + H + (0 if cfg.tie_word_embeddings else V * H)
    per_layer = F * H + F + H * H + H + 2 * H + H * I + I + I * H + H + 2 * H
    emb = V * H + cfg.max_position_embeddings * H + 2 * H
    dec = (0 if cfg.tie_word_embeddings else V * H) + V
    return L * per_layer + emb + dec


def gpt_train_flops(batch_size: int, seq_len: int, cfg: GPTConfig, backward: bool = True,
                    checkpoint_activations: bool = False) -> float:
    """The reference's FLOP accounting verbatim (alpa/util.py:1658-1687)."""
    factor = 24 + (48 if backward else 0) + (24 if checkpoint_activations else 0)
    H, L, V = cfg.hidden_size, cfg.num_hidden_layers, cfg.vocab_size
    return (factor * batch_size * seq_len * H * H * L * (1 + seq_len / (6 * H)) +
            6 * batch_size * seq_len * H * V)


# ---- Hugging Face Llama checkpoints
def llama_config_from_hf(hf_config, **kw) -> GPTConfig:
    """The GPTConfig(arch="llama") of a transformers LlamaConfig (causal, RMSNorm eps and rope theta taken over);
    `kw` overrides or adds fields (dtype, pipeline markers, ...).  Raises ValueError for a checkpoint this model does not
    compute: rope scaling, attention / MLP biases, a head dim other than H / heads, an activation other than SiLU, or a
    sliding window."""
    c = hf_config
    # transformers >= 5 keeps theta and any scaling in rope_parameters (rope_scaling is an alias); older releases keep
    # rope_theta apart and set rope_scaling only when the frequencies are scaled
    rope = dict(getattr(c, "rope_parameters", None) or getattr(c, "rope_scaling", None) or {})
    if rope.get("rope_type", rope.get("type", "default")) != "default":
        raise ValueError(f"rope scaling is not supported: {rope}")
    if getattr(c, "attention_bias", False) or getattr(c, "mlp_bias", False):
        raise ValueError("attention_bias / mlp_bias are not supported")
    H, nh = c.hidden_size, c.num_attention_heads
    if getattr(c, "head_dim", None) not in (None, H // nh):
        raise ValueError(f"head_dim {c.head_dim} != hidden_size / num_attention_heads = {H // nh}")
    if getattr(c, "hidden_act", "silu") != "silu":
        raise ValueError(f"hidden_act {c.hidden_act!r} is not supported (SiLU only)")
    if getattr(c, "sliding_window", None) or getattr(c, "use_sliding_window", False):
        raise ValueError("sliding-window attention is not supported")
    theta = rope.get("rope_theta", getattr(c, "rope_theta", 10000.0))
    args = dict(arch="llama", vocab_size=c.vocab_size, hidden_size=H, num_hidden_layers=c.num_hidden_layers,
                num_attention_heads=nh, num_key_value_heads=getattr(c, "num_key_value_heads", None) or nh,
                intermediate_size=c.intermediate_size, max_position_embeddings=c.max_position_embeddings,
                layer_norm_eps=c.rms_norm_eps, initializer_range=getattr(c, "initializer_range", 0.02), causal=True,
                tie_word_embeddings=bool(getattr(c, "tie_word_embeddings", False)), rope_theta=float(theta))
    args.update(kw)
    return GPTConfig(**args)


def pack_llama_qkv(q, k, v, kv_heads: int):
    """The fused QKV rows: for each K/V head, the q rows of its G query heads, then its k rows, then its v rows.
    q: [heads * D, X], k / v: [kv_heads * D, X], for any row width X (a weight, or a LoRA B)."""
    X = q.shape[-1]
    return torch.cat([t.reshape(kv_heads, -1, X) for t in (q, k, v)], 1).reshape(-1, X)


def pack_llama_fc1(gate, up):
    """fc1's rows: gate_proj and up_proj rows interleaved.  gate / up: [I, X] -> [2 I, X]."""
    return torch.stack([gate, up], 1).reshape(2 * gate.shape[0], gate.shape[-1])


def llama_params_from_hf(state_dict, cfg: GPTConfig) -> dict:
    """GPTModel(cfg) parameters (arch="llama", cast to cfg.dtype) from a LlamaForCausalLM state dict.  The fused QKV
    weight takes, for each K/V head, the q_proj rows of its G query heads, then its k_proj rows, then its v_proj rows;
    fc1 interleaves gate_proj and up_proj rows."""
    sd = {k[len("model."):] if k.startswith("model.") else k: v for k, v in state_dict.items()}
    kv = cfg.num_key_value_heads or cfg.num_attention_heads
    out = {"wte": sd["embed_tokens.weight"], "ln_f_g": sd["norm.weight"]}
    if not cfg.tie_word_embeddings:
        out["decoder_w"] = sd["lm_head.weight"]
    for i in range(cfg.num_hidden_layers):
        p, a, m = f"layers.{i}.", f"layers.{i}.self_attn.", f"layers.{i}.mlp."
        b = f"blocks.{i}."
        out[b + "qkv_w"] = pack_llama_qkv(sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"], kv)
        out[b + "proj_w"] = sd[a + "o_proj.weight"]
        out[b + "ln1_g"] = sd[p + "input_layernorm.weight"]
        out[b + "ln2_g"] = sd[p + "post_attention_layernorm.weight"]
        out[b + "fc1_w"] = pack_llama_fc1(sd[m + "gate_proj.weight"], sd[m + "up_proj.weight"])
        out[b + "fc2_w"] = sd[m + "down_proj.weight"]
    return {k: v.detach().to(cfg.dtype).contiguous() for k, v in out.items()}
