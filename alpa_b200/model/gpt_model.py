"""GPT language model built from the alpa_b200 primitives.

Architecture parity with the reference's benchmark model (alpa/model/gpt_model.py:19-93 on top of
alpa/model/bert_model.py: word+position embeddings -> LayerNorm -> L x [self-attention, dense,
residual+LayerNorm, dense+GELU, dense, residual+LayerNorm] (post-LN) -> vocabulary projection + bias).
The reference attends bidirectionally with an all-ones mask in its GPT benchmark
(benchmark_one_case_gpt_bert.py:142-148); `causal=True` gives the usual decoder masking.

H100 mapping: fused QKV projection (features ordered (head, {q,k,v}, D) so tensor-parallel splits are
head splits; with grouped-query attention (K/V head, {G query heads, k, v}, D)), packed flash attention, GELU / bias / pre-activation fused into GEMM epilogues,
residual-add fused into LayerNorm, per-token fused cross-entropy.
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
    causal: bool = False                       # reference benchmark: bidirectional + all-ones mask
    tie_word_embeddings: bool = False
    add_manual_pipeline_markers: bool = False  # mark a layer boundary every `pipeline_mp_size` blocks
    pipeline_mp_size: int = 0
    gradient_checkpointing: bool = False
    hidden_dropout_prob: float = 0.0           # counter-based dropout (ops.dropout) after proj / fc2 when a seed is passed
    dtype: torch.dtype = torch.bfloat16

    def __post_init__(self):
        if self.intermediate_size is None:
            self.intermediate_size = 4 * self.hidden_size
        assert self.hidden_size % self.num_attention_heads == 0
        kv = self.num_key_value_heads
        assert kv is None or (kv > 0 and self.num_attention_heads % kv == 0), \
            "num_key_value_heads must divide num_attention_heads"

    @property
    def grouped_query(self) -> bool:
        return self.num_key_value_heads not in (None, self.num_attention_heads)

    @property
    def qkv_features(self) -> int:
        """Output features of the fused QKV projection: 3 H, or (G + 2) Hkv D with grouped-query attention."""
        if not self.grouped_query:
            return 3 * self.hidden_size
        return (self.num_attention_heads + 2 * self.num_key_value_heads) * (self.hidden_size // self.num_attention_heads)


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
        if cfg.grouped_query:
            # features ordered (K/V head, {its G query heads, k, v}, D): a column split is a split over K/V heads
            kvh = cfg.num_key_value_heads
            qkv = ops.linear(x, self.qkv_w, self.qkv_b).view(B, S, kvh, nh // kvh + 2, D)
            o, _ = ops.attention_gqa_packed(qkv, 1.0 / math.sqrt(D), cfg.causal)
        else:
            qkv = ops.linear(x, self.qkv_w, self.qkv_b).view(B, S, nh, 3, D)
            o, _ = ops.attention_qkvpacked(qkv, 1.0 / math.sqrt(D), cfg.causal)
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


class GPTModel(nn.Module):
    """`forward(input_ids, position_ids) -> logits [B, S, V]`."""

    def __init__(self, cfg: GPTConfig, device=None):
        super().__init__()
        self.cfg = cfg
        kw = dict(device=device, dtype=cfg.dtype)
        std = cfg.initializer_range
        H = cfg.hidden_size
        self.wte = nn.Parameter(torch.randn(cfg.vocab_size, H, **kw) * std)
        self.wpe = nn.Parameter(torch.randn(cfg.max_position_embeddings, H, **kw) * std)
        self.emb_ln_g = nn.Parameter(torch.ones(H, **kw))
        self.emb_ln_b = nn.Parameter(torch.zeros(H, **kw))
        self.blocks = nn.ModuleList([GPTBlock(cfg, device) for _ in range(cfg.num_hidden_layers)])
        if not cfg.tie_word_embeddings:
            self.decoder_w = nn.Parameter(torch.randn(cfg.vocab_size, H, **kw) * std)
        self.decoder_b = nn.Parameter(torch.zeros(cfg.vocab_size, **kw))

    def hidden_states(self, input_ids, position_ids, dropout_seed=None):
        cfg = self.cfg
        x = ops.embedding(input_ids, self.wte) + ops.embedding(position_ids, self.wpe)
        x, _, _ = ops.layer_norm(x, self.emb_ln_g, self.emb_ln_b, cfg.layer_norm_eps)
        if dropout_seed is not None and cfg.hidden_dropout_prob > 0.0:
            x = ops.dropout_like(x, cfg.hidden_dropout_prob, dropout_seed, stream=0)
        for i, blk in enumerate(self.blocks):
            if cfg.add_manual_pipeline_markers and cfg.pipeline_mp_size > 1 and i > 0:
                per = max(1, cfg.num_hidden_layers // cfg.pipeline_mp_size)
                if i % per == 0 and i // per < cfg.pipeline_mp_size:
                    x = mark_pipeline_boundary(x)
            x = blk(x, dropout_seed, i) if dropout_seed is not None else blk(x)
        return x

    def forward(self, input_ids, position_ids, dropout_seed=None):
        """`dropout_seed`: int64 scalar tensor (e.g. from the step counter) enables hidden-state dropout in training."""
        x = self.hidden_states(input_ids, position_ids, dropout_seed)
        w = self.wte if self.cfg.tie_word_embeddings else self.decoder_w
        return ops.linear(x, w, self.decoder_b)


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
