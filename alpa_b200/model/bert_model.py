"""BERT (encoder-only transformer) built from the alpa_b200 primitives.

Reference: alpa/model/bert_model.py (BertConfig:27, FlaxBertEmbeddings:110, FlaxBertSelfAttention:158,
FlaxBertLayer:338, FlaxBertLayerCollection:380, FlaxBertEncoder:437, FlaxBertPooler:461, FlaxBertLMPredictionHead:
497, FlaxBertForPreTraining / ForMaskedLM / ForSequenceClassification :556-884).  Same post-LN architecture; the
encoder layer is `GPTBlock` (fused QKV GEMM, packed flash attention, GELU in the GEMM epilogue, residual fused into
LayerNorm).  A padding mask disables the flash kernel for that call (the sm_90a attention kernel supports full and
causal masks); padded batches run the composed softmax path with identical maths.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from alpa_b200 import ops
from alpa_b200.model.gpt_model import GPTBlock, GPTConfig
from alpa_b200.parallel.pipeline.primitive_def import mark_pipeline_boundary


@dataclass
class BertConfig(GPTConfig):
    vocab_size: int = 30522
    max_position_embeddings: int = 512
    type_vocab_size: int = 2
    num_labels: int = 2
    hidden_dropout_prob: float = 0.0          # the reference benchmarks run without dropout
    tie_word_embeddings: bool = True


class BertEmbeddings(nn.Module):
    def __init__(self, cfg: BertConfig, device=None):
        super().__init__()
        kw = dict(device=device, dtype=cfg.dtype)
        H, std = cfg.hidden_size, cfg.initializer_range
        self.cfg = cfg
        self.word = nn.Parameter(torch.randn(cfg.vocab_size, H, **kw) * std)
        self.position = nn.Parameter(torch.randn(cfg.max_position_embeddings, H, **kw) * std)
        self.token_type = nn.Parameter(torch.randn(cfg.type_vocab_size, H, **kw) * std)
        self.ln_g = nn.Parameter(torch.ones(H, **kw))
        self.ln_b = nn.Parameter(torch.zeros(H, **kw))

    def forward(self, input_ids, token_type_ids, position_ids):
        x = ops.embedding(input_ids, self.word) + ops.embedding(position_ids, self.position) \
            + ops.embedding(token_type_ids, self.token_type)
        x, _, _ = ops.layer_norm(x, self.ln_g, self.ln_b, self.cfg.layer_norm_eps)
        return x


class BertLayer(GPTBlock):
    """Encoder layer; with a padding mask the attention core is the composed (masked softmax) path."""

    def forward(self, x, attention_mask: Optional[torch.Tensor] = None):
        if attention_mask is None:
            return super().forward(x)
        cfg = self.cfg
        B, S, H = x.shape
        nh = cfg.num_attention_heads
        D = H // nh
        qkv = ops.linear(x, self.qkv_w, self.qkv_b).view(B, S, nh, 3, D)
        q, k, v = qkv[:, :, :, 0].transpose(1, 2), qkv[:, :, :, 1].transpose(1, 2), qkv[:, :, :, 2].transpose(1, 2)
        bias = (1.0 - attention_mask[:, None, None, :].to(torch.float32)) * -1e9
        p = torch.softmax((q @ k.transpose(-1, -2)).float() / math.sqrt(D) + bias, dim=-1).to(x.dtype)
        o = (p @ v).transpose(1, 2).reshape(B, S, H)
        a = ops.linear(o, self.proj_w, self.proj_b)
        x1, _, _, _ = ops.add_layer_norm(a, x, self.ln1_g, self.ln1_b, cfg.layer_norm_eps)
        h, _ = ops.linear_act(x1, self.fc1_w, self.fc1_b, "gelu")
        m = ops.linear(h, self.fc2_w, self.fc2_b)
        x2, _, _, _ = ops.add_layer_norm(m, x1, self.ln2_g, self.ln2_b, cfg.layer_norm_eps)
        return x2


class BertModel(nn.Module):
    """-> (sequence_output [B,S,H], pooled_output [B,H] or None)"""

    def __init__(self, cfg: BertConfig, add_pooling_layer: bool = True, device=None):
        super().__init__()
        self.cfg = cfg
        kw = dict(device=device, dtype=cfg.dtype)
        H, std = cfg.hidden_size, cfg.initializer_range
        self.embeddings = BertEmbeddings(cfg, device)
        self.layers = nn.ModuleList([BertLayer(cfg, device) for _ in range(cfg.num_hidden_layers)])
        self.add_pooling_layer = add_pooling_layer
        if add_pooling_layer:
            self.pool_w = nn.Parameter(torch.randn(H, H, **kw) * std)
            self.pool_b = nn.Parameter(torch.zeros(H, **kw))

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, position_ids=None):
        cfg = self.cfg
        B, S = input_ids.shape
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        if position_ids is None:
            position_ids = torch.arange(S, device=input_ids.device).unsqueeze(0).expand(B, S)
        x = self.embeddings(input_ids, token_type_ids, position_ids)
        for i, layer in enumerate(self.layers):
            if cfg.add_manual_pipeline_markers and cfg.pipeline_mp_size > 1 and i > 0:
                per = max(1, cfg.num_hidden_layers // cfg.pipeline_mp_size)
                if i % per == 0 and i // per < cfg.pipeline_mp_size:
                    x = mark_pipeline_boundary(x)
            x = layer(x, attention_mask)
        pooled = None
        if self.add_pooling_layer:
            pooled = torch.tanh(ops.linear(x[:, 0], self.pool_w, self.pool_b))
        return x, pooled


class BertLMPredictionHead(nn.Module):
    """dense + GELU + LayerNorm + (tied) decoder (reference: FlaxBertLMPredictionHead:497)."""

    def __init__(self, cfg: BertConfig, device=None):
        super().__init__()
        kw = dict(device=device, dtype=cfg.dtype)
        H, std = cfg.hidden_size, cfg.initializer_range
        self.cfg = cfg
        self.transform_w = nn.Parameter(torch.randn(H, H, **kw) * std)
        self.transform_b = nn.Parameter(torch.zeros(H, **kw))
        self.ln_g = nn.Parameter(torch.ones(H, **kw))
        self.ln_b = nn.Parameter(torch.zeros(H, **kw))
        if not cfg.tie_word_embeddings:
            self.decoder_w = nn.Parameter(torch.randn(cfg.vocab_size, H, **kw) * std)
        self.decoder_b = nn.Parameter(torch.zeros(cfg.vocab_size, **kw))

    def forward(self, x, shared_embedding=None):
        h, _ = ops.linear_act(x, self.transform_w, self.transform_b, "gelu")
        h, _, _ = ops.layer_norm(h, self.ln_g, self.ln_b, self.cfg.layer_norm_eps)
        w = shared_embedding if self.cfg.tie_word_embeddings else self.decoder_w
        return ops.linear(h, w, self.decoder_b)


class BertForMaskedLM(nn.Module):
    def __init__(self, cfg: BertConfig, device=None):
        super().__init__()
        self.cfg = cfg
        self.bert = BertModel(cfg, add_pooling_layer=False, device=device)
        self.cls = BertLMPredictionHead(cfg, device)

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, position_ids=None):
        x, _ = self.bert(input_ids, attention_mask, token_type_ids, position_ids)
        return self.cls(x, self.bert.embeddings.word)


class BertForPreTraining(nn.Module):
    """MLM logits + next-sentence logits (reference: FlaxBertForPreTrainingModule:556)."""

    def __init__(self, cfg: BertConfig, device=None):
        super().__init__()
        kw = dict(device=device, dtype=cfg.dtype)
        self.cfg = cfg
        self.bert = BertModel(cfg, add_pooling_layer=True, device=device)
        self.cls = BertLMPredictionHead(cfg, device)
        self.nsp_w = nn.Parameter(torch.randn(8, cfg.hidden_size, **kw) * cfg.initializer_range)  # 2 classes, padded to 8
        self.nsp_b = nn.Parameter(torch.zeros(8, **kw))

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, position_ids=None):
        x, pooled = self.bert(input_ids, attention_mask, token_type_ids, position_ids)
        return self.cls(x, self.bert.embeddings.word), ops.linear(pooled, self.nsp_w, self.nsp_b)[:, :2]


class BertForSequenceClassification(nn.Module):
    def __init__(self, cfg: BertConfig, device=None):
        super().__init__()
        kw = dict(device=device, dtype=cfg.dtype)
        self.cfg = cfg
        self.bert = BertModel(cfg, add_pooling_layer=True, device=device)
        n = (cfg.num_labels + 7) // 8 * 8      # GEMM N must be a multiple of 8; extra logits are sliced off
        self.cls_w = nn.Parameter(torch.randn(n, cfg.hidden_size, **kw) * cfg.initializer_range)
        self.cls_b = nn.Parameter(torch.zeros(n, **kw))

    def forward(self, input_ids, attention_mask=None, token_type_ids=None, position_ids=None):
        _, pooled = self.bert(input_ids, attention_mask, token_type_ids, position_ids)
        return ops.linear(pooled, self.cls_w, self.cls_b)[:, :self.cfg.num_labels]


def bert_mlm_loss(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """Mean CE over positions with label >= 0... the reference masks with label > 0
    (benchmark_one_case_gpt_bert.py:106-110)."""
    V = logits.shape[-1]
    loss, _ = ops.cross_entropy(logits.reshape(-1, V), labels.reshape(-1).clamp(min=0))
    mask = (labels.reshape(-1) > 0).to(loss.dtype)
    return (loss * mask).sum() / mask.sum().clamp(min=1.0)


# (S, H, L, heads, V) -- reference benchmark/alpa/suite_manual_gpt.py uses the GPT table for BERT as well
BERT_SPECS = {
    "base": (512, 768, 12, 12, 30522),
    "large": (512, 1024, 24, 16, 30522),
}
