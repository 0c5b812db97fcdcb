"""Vision Transformer for image classification.

Reference: examples/ViT/run_image_classification.py fine-tunes HuggingFace's FlaxViTForImageClassification under
alpa.parallelize; the model itself comes from `transformers`.  Here the encoder is built from the framework's own
fused transformer block (alpa_b200.model.gpt_model.GPTBlock: wgmma GEMMs with fused bias/GELU epilogues, flash
attention, fused add+LayerNorm), so every ViT matmul runs on the sm_90a kernels and the auto-sharding planner sees
the same operator set as for GPT/BERT.  Patch embedding is the strided convolution written as unfold + GEMM.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn

from alpa_b200 import ops
from alpa_b200.model.gpt_model import GPTBlock, GPTConfig
from alpa_b200.parallel.pipeline.primitive_def import mark_pipeline_boundary


@dataclass
class ViTConfig(GPTConfig):
    image_size: int = 224
    patch_size: int = 16
    num_channels: int = 3
    num_labels: int = 1000
    vocab_size: int = 0
    causal: bool = False
    layer_norm_eps: float = 1e-6

    @property
    def num_patches(self) -> int:
        return (self.image_size // self.patch_size) ** 2


# name -> (hidden, layers, heads, mlp) (the ViT paper's B/L/H sizes used by google/vit-* checkpoints)
VIT_SPECS = {"tiny": (192, 12, 3, 768), "small": (384, 12, 6, 1536), "base": (768, 12, 12, 3072),
             "large": (1024, 24, 16, 4096), "huge": (1280, 32, 16, 5120)}


def vit_config(name: str, **kw) -> ViTConfig:
    h, l, nh, mlp = VIT_SPECS[name]
    return ViTConfig(hidden_size=h, num_hidden_layers=l, num_attention_heads=nh, intermediate_size=mlp, **kw)


class ViTModel(nn.Module):
    """`forward(pixel_values [B, C, H, W]) -> logits [B, num_labels]`"""

    def __init__(self, cfg: ViTConfig, device=None):
        super().__init__()
        self.cfg = cfg
        kw = dict(device=device, dtype=cfg.dtype)
        H, std = cfg.hidden_size, cfg.initializer_range
        pdim = cfg.num_channels * cfg.patch_size ** 2
        self.patch_w = nn.Parameter(torch.randn(H, pdim, **kw) * std)
        self.patch_b = nn.Parameter(torch.zeros(H, **kw))
        self.cls_token = nn.Parameter(torch.zeros(1, 1, H, **kw))
        self.pos_emb = nn.Parameter(torch.randn(1, cfg.num_patches + 1, H, **kw) * std)
        self.blocks = nn.ModuleList([GPTBlock(cfg, device) for _ in range(cfg.num_hidden_layers)])
        self.ln_g = nn.Parameter(torch.ones(H, **kw))
        self.ln_b = nn.Parameter(torch.zeros(H, **kw))
        self.head_w = nn.Parameter(torch.randn(cfg.num_labels, H, **kw) * std)
        self.head_b = nn.Parameter(torch.zeros(cfg.num_labels, **kw))

    def patchify(self, pixel_values: torch.Tensor) -> torch.Tensor:
        cfg = self.cfg
        B, C, Hh, Ww = pixel_values.shape
        p = cfg.patch_size
        x = pixel_values.reshape(B, C, Hh // p, p, Ww // p, p).permute(0, 2, 4, 1, 3, 5)
        return x.reshape(B, (Hh // p) * (Ww // p), C * p * p)

    def forward(self, pixel_values):
        cfg = self.cfg
        B = pixel_values.shape[0]
        x = ops.linear(self.patchify(pixel_values).to(cfg.dtype), self.patch_w, self.patch_b)
        x = torch.cat([self.cls_token.expand(B, 1, -1), x], dim=1) + self.pos_emb
        for i, blk in enumerate(self.blocks):
            if cfg.add_manual_pipeline_markers and cfg.pipeline_mp_size > 1 and i > 0:
                per = max(1, cfg.num_hidden_layers // cfg.pipeline_mp_size)
                if i % per == 0 and i // per < cfg.pipeline_mp_size:
                    x = mark_pipeline_boundary(x)
            x = blk(x)
        cls, _, _ = ops.layer_norm(x[:, 0].contiguous(), self.ln_g, self.ln_b, cfg.layer_norm_eps)
        return ops.linear(cls, self.head_w, self.head_b)


def classification_loss(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    return torch.nn.functional.cross_entropy(logits.float(), labels)
