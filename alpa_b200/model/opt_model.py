"""Decoder-only LMs for serving: OPT, BLOOM, CodeGen and Llama variants of one tensor-parallel transformer.

Reference: examples/llm_serving/model/opt_model.py (OPTConfig:44, OPTEmbeddings:95, OPTSelfAttention:138 with the
KV cache threaded through `attention_cache`, OPTTransformerLayer:316, OPTForLMModule:470, get_opt_config:533,
init_cache_np:756, load_params_np:875), bloom_model.py, codegen_model.py.  The reference compiles prompt ("encoder",
chunked) and single-token ("decoder") executables with alpa's pipeshard runtime.

H100 design: a dedicated SPMD inference engine -- one process per GPU, Megatron tensor parallelism written out
explicitly (column-parallel QKV / FC1, row-parallel out-proj / FC2, vocab-parallel embedding and LM head), the
all-reduces on the NVSwitch (NCCL / NVLS), KV cache resident in HBM as [B, S_max, heads_local, D] per layer, the
prompt phase on the flash-attention kernel and every decode step replayed from a CUDA graph.  Weights can be kept in
fp8 (e4m3, per-output-channel scales) to halve the weight traffic that bounds decode, and the KV cache in fp8
(`kv_cache_dtype="fp8"`: e4m3 rows with one scale per token and head, `ops.Fp8KV`) to halve the cache traffic that
bounds decode at long contexts and large batches.

`arch="llama"` serves the Llama-style model of `gpt_model.GPTModel(arch="llama")` from its parameters: pre-RMSNorm
blocks without biases, grouped-query attention with rotary embeddings, a SwiGLU MLP.  Its KV cache holds only the K/V
heads ([B, S_max, Hkv_local, D]); a decode step rotates, appends and attends in one kernel that reads each K/V row once
for its whole group of query heads.
"""
from __future__ import annotations

import math
import re
import weakref
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F

from alpa_b200 import ops
from alpa_b200.model.gpt_model import pack_llama_fc1, pack_llama_qkv


@dataclass
class OPTConfig:
    """(reference: OPTConfig, opt_model.py:44-77; bloom/codegen configs share the fields)"""
    arch: str = "opt"                     # opt | bloom | codegen | llama
    vocab_size: int = 50272
    hidden_size: int = 768
    num_hidden_layers: int = 12
    num_attention_heads: int = 12
    ffn_dim: int = 3072
    max_position_embeddings: int = 2048
    layer_norm_eps: float = 1e-5
    pad_token_id: int = 1
    activation: str = "relu"              # opt: relu, bloom/codegen: gelu
    rotary_dim: int = 0                   # codegen
    # codegen (GPT-J layout): one LayerNorm per block feeding attention and MLP in parallel, no attention biases,
    # an untied LM head with a bias.  None = follow `arch`.
    parallel_block: Optional[bool] = None
    tie_word_embeddings: Optional[bool] = None
    dtype: torch.dtype = torch.bfloat16
    weight_dtype: str = "bf16"            # bf16 | fp8 (e4m3 weights, per-channel scales) | mxfp8 (e4m3 + UE8M0 per 32)
    # llama: K/V heads of grouped-query attention (None = num_attention_heads) and the rotary base; layer_norm_eps is
    # the RMSNorm eps and ffn_dim the SwiGLU width
    num_key_value_heads: Optional[int] = None
    rope_theta: float = 10000.0
    # bf16 | fp8: e4m3 K/V rows with one fp32 scale per (token, K/V head) (ops.Fp8KV), about half the cache bytes
    kv_cache_dtype: str = "bf16"
    # multi-LoRA serving: adapter slots (0 = off: nothing is allocated) and the largest rank an adapter may have
    max_loras: int = 0
    max_lora_rank: int = 16

    def __post_init__(self):
        if self.kv_cache_dtype not in ("bf16", "fp8"):
            raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8', not {self.kv_cache_dtype!r}")
        if self.max_loras < 0 or not 1 <= self.max_lora_rank <= 64:
            raise ValueError("need max_loras >= 0 and 1 <= max_lora_rank <= 64")
        if self.parallel_block is None:
            self.parallel_block = self.arch == "codegen"
        if self.tie_word_embeddings is None:
            self.tie_word_embeddings = self.arch not in ("codegen", "llama")
        if self.num_attention_heads % self.kv_heads:
            raise ValueError("num_key_value_heads must divide num_attention_heads")
        if self.arch != "llama" and self.kv_heads != self.num_attention_heads:
            raise ValueError(f"grouped-query attention is served for arch='llama' only, not {self.arch!r}")

    @property
    def kv_heads(self):
        return self.num_key_value_heads or self.num_attention_heads

    @property
    def head_dim(self):
        return self.hidden_size // self.num_attention_heads


# name -> (layers, hidden, heads) (reference: get_opt_config, opt_model.py:533-640)
OPT_SPECS = {
    "125m": (12, 768, 12), "350m": (24, 1024, 16), "1.3b": (24, 2048, 32), "2.7b": (32, 2560, 32),
    "6.7b": (32, 4096, 32), "13b": (40, 5120, 40), "30b": (48, 7168, 56), "66b": (64, 9216, 72),
    "175b": (96, 12288, 96),
}
BLOOM_SPECS = {"560m": (24, 1024, 16), "1b7": (24, 2048, 16), "3b": (30, 2560, 32), "7b1": (30, 4096, 32),
               "176b": (70, 14336, 112)}
CODEGEN_SPECS = {"350m": (20, 1024, 16), "2b": (32, 2560, 32), "6b": (33, 4096, 16), "16b": (34, 6144, 24)}
CODEGEN_ROTARY = {"350m": 32, "2b": 64, "6b": 64, "16b": 64}          # (reference: codegen_model.py:514-537)
# name -> (layers, hidden, heads, kv heads, ffn, vocab, rope theta, max positions) of the Hugging Face configs
LLAMA_SPECS = {"2-7b": (32, 4096, 32, 32, 11008, 32000, 10000.0, 4096),
               "2-70b": (80, 8192, 64, 8, 28672, 32000, 10000.0, 4096),
               "3-8b": (32, 4096, 32, 8, 14336, 128256, 500000.0, 8192)}


def get_config(name: str, **kw) -> OPTConfig:
    """'opt-2.7b', 'bloom-7b1', 'codegen-2b', 'llama-3-8b' ... (reference: get_opt_config / get_bloom_config /
    get_codegen_config)"""
    fam, _, size = name.lower().replace("facebook/", "").replace("alpa/", "").replace("meta-llama/", "").partition("-")
    if fam == "llama":
        L, H, nh, kv, I, V, theta, S = LLAMA_SPECS[size.replace("llama-", "").removesuffix("-hf")]
        return OPTConfig(arch="llama", vocab_size=V, hidden_size=H, num_hidden_layers=L, num_attention_heads=nh,
                         num_key_value_heads=kv, ffn_dim=I, max_position_embeddings=S, rope_theta=theta,
                         pad_token_id=0, activation="silu", **kw)
    if fam == "opt":
        L, H, nh = OPT_SPECS[size]
        return OPTConfig(arch="opt", vocab_size=50272, hidden_size=H, num_hidden_layers=L, num_attention_heads=nh,
                         ffn_dim=4 * H, **kw)
    if fam == "bloom":
        L, H, nh = BLOOM_SPECS[size]
        return OPTConfig(arch="bloom", vocab_size=250880, hidden_size=H, num_hidden_layers=L, num_attention_heads=nh,
                         ffn_dim=4 * H, activation="gelu", **kw)
    if fam == "codegen":
        size = size.split("-")[0]                               # "codegen-2b-mono" / "-multi" / "-nl": same shapes
        L, H, nh = CODEGEN_SPECS[size]
        return OPTConfig(arch="codegen", vocab_size=51200, hidden_size=H, num_hidden_layers=L, num_attention_heads=nh,
                         ffn_dim=4 * H, activation="gelu", rotary_dim=CODEGEN_ROTARY[size], **kw)
    raise ValueError(name)


def serving_config_from_gpt(gcfg, **kw) -> OPTConfig:
    """The serving config of a `GPTConfig(arch="llama")` (e.g. from `llama_config_from_hf`); `kw` overrides fields
    (dtype, weight_dtype, ...)."""
    if gcfg.arch != "llama":
        raise ValueError(f"only arch='llama' GPT configs are served, not {gcfg.arch!r}")
    args = dict(arch="llama", vocab_size=gcfg.vocab_size, hidden_size=gcfg.hidden_size,
                num_hidden_layers=gcfg.num_hidden_layers, num_attention_heads=gcfg.num_attention_heads,
                num_key_value_heads=gcfg.num_key_value_heads or gcfg.num_attention_heads,
                ffn_dim=gcfg.intermediate_size, max_position_embeddings=gcfg.max_position_embeddings,
                layer_norm_eps=gcfg.layer_norm_eps, pad_token_id=0, activation="silu",
                tie_word_embeddings=gcfg.tie_word_embeddings, rope_theta=gcfg.rope_theta, dtype=gcfg.dtype)
    args.update(kw)
    return OPTConfig(**args)


def gpt_config_from_serving(cfg: OPTConfig):
    """The `GPTConfig(arch="llama")` whose parameter layout `DecoderLM(cfg)` takes."""
    from alpa_b200.model.gpt_model import GPTConfig
    return GPTConfig(arch="llama", vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size,
                     num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                     num_key_value_heads=cfg.num_key_value_heads, intermediate_size=cfg.ffn_dim,
                     max_position_embeddings=cfg.max_position_embeddings, layer_norm_eps=cfg.layer_norm_eps,
                     tie_word_embeddings=cfg.tie_word_embeddings, rope_theta=cfg.rope_theta, dtype=cfg.dtype)


class _TPLinear:
    """y = x W^T (+b).  W is this rank's slice ([N_local, K] column-parallel or [N, K_local] row-parallel); stored bf16
    or fp8 e4m3 with one fp32 scale per output channel."""

    def __init__(self, w: torch.Tensor, b: Optional[torch.Tensor], fp8):
        self.b = b
        self.mx = fp8 == "mxfp8"
        self.fp8 = fp8 = bool(fp8) and not self.mx
        if self.mx:
            # OCP microscaling: e4m3 elements, one power-of-two scale per 32 input channels, stored in the scale-atom
            # layout read by the MXFP8 GEMM (opt-in: the kernel has not had a hardware run yet)
            self.w, self.scale = ops.quantize_mxfp8(w.contiguous())
        elif fp8:
            amax = w.float().abs().amax(dim=1).clamp(min=1e-8)
            self.scale = (amax / 448.0).to(torch.float32)
            self.w = (w.float() / self.scale[:, None]).to(torch.float8_e4m3fn)
        else:
            self.w = w
            self.scale = None

    def __call__(self, x: torch.Tensor, act: str = "none", residual: Optional[torch.Tensor] = None,
                 ln=None) -> torch.Tensor:
        """`ln` = (gamma, beta, eps) or ops.RMSNormArgs(gamma, eps): normalise x first (fused into the decode GEMV's
        prologue)."""
        rows = x.numel() // x.shape[-1]
        if self.mx:
            if ln is not None:
                x = ops.fast.norm_rows(x, ln)
            y = ops.fast.linear_mxfp8(x, self.w, self.scale, self.b, act)
            return y if residual is None else y + residual
        if rows <= 8 and x.is_cuda and x.dtype == torch.bfloat16:
            # decode: weight-streaming GEMV (no activation quantisation, no tile padding), LN / residual fused
            return ops.fast.linear_decode(x, self.w, self.scale, self.b, act, residual, ln)
        if ln is not None:
            x = ops.fast.norm_rows(x, ln)
        if residual is not None:
            return self(x, act) + residual
        if self.fp8:
            return ops.fast.linear_fp8(x, self.w, self.scale, self.b, act)
        if act == "none":
            return ops.fast.linear(x, self.w, self.b)
        return ops.fast.linear_act(x, self.w, self.b, act)[0]

    def nbytes(self):
        return self.w.numel() * self.w.element_size()


# LoRA targets per architecture: the PEFT module name -> (DecoderLM projection, its part of the stacked rank).  OPT's
# fc1 is no target: its activation is fused into the GEMM epilogue, and the delta would have to go in before it.
LORA_TARGETS = {
    "llama": {"q_proj": ("qkv", 0), "k_proj": ("qkv", 1), "v_proj": ("qkv", 2), "o_proj": ("out", 0),
              "gate_proj": ("fc1", 0), "up_proj": ("fc1", 1), "down_proj": ("fc2", 0)},
    "opt": {"q_proj": ("qkv", 0), "k_proj": ("qkv", 1), "v_proj": ("qkv", 2), "out_proj": ("out", 0),
            "fc2": ("fc2", 0)},
}
# PEFT tensor names: `base_model.model.model.layers.3.self_attn.q_proj.lora_A.weight`, `...decoder.layers.3.fc2.lora_B
# .weight`
_LORA_NAME = re.compile(r"layers\.(\d+)\.(?:\w+\.)?(\w+)\.lora_([AB])(?:\.weight)?$")


def _alibi_slopes(n: int) -> torch.Tensor:
    def pow2(k):
        start = 2 ** (-2 ** -(math.log2(k) - 3))
        return [start * (start ** i) for i in range(k)]
    if math.log2(n).is_integer():
        return torch.tensor(pow2(n))
    k = 2 ** math.floor(math.log2(n))
    return torch.tensor(pow2(k) + pow2(2 * k)[0::2][:n - k])


def _oneshot_flags(group):
    """Symmetric flag pad of the one-shot all-reduce (one uint32 per peer)."""
    from alpa_b200.collective.fused import SymmWorkspace
    return SymmWorkspace(group, 1024)


class DecoderLM:
    """Tensor-parallel decoder with a KV cache.  `group` = the TP process group (None = single GPU)."""

    def __init__(self, cfg: OPTConfig, device="cuda", group=None, seed: int = 0, params: Optional[Dict] = None):
        self.cfg = cfg
        self.device = torch.device(device)
        self.group = group
        self.tp = dist.get_world_size(group) if group is not None else 1
        self.rank = dist.get_rank(group) if group is not None else 0
        H, I, nh, V = cfg.hidden_size, cfg.ffn_dim, cfg.num_attention_heads, cfg.vocab_size
        if cfg.arch == "llama" and cfg.kv_heads % self.tp:
            raise ValueError(f"tensor parallelism over {self.tp} ranks needs num_key_value_heads "
                             f"({cfg.kv_heads}) to be a multiple of it")
        assert nh % self.tp == 0 and I % self.tp == 0
        self.nh_local = nh // self.tp
        self.kv_local = cfg.kv_heads // self.tp           # K/V heads of this rank (= nh_local but for GQA)
        self.D = cfg.head_dim
        self.Vp = (V + 8 * self.tp - 1) // (8 * self.tp) * (8 * self.tp)      # padded so every shard is a multiple of 8
        self.V_local = self.Vp // self.tp
        fp8 = "mxfp8" if cfg.weight_dtype == "mxfp8" else cfg.weight_dtype == "fp8"
        g = torch.Generator(device="cpu").manual_seed(seed)          # identical full weights on every rank, then sliced

        def rnd(*shape, std=0.02):
            if params is not None:
                raise KeyError
            return (torch.randn(*shape, generator=g) * std).to(cfg.dtype)

        def get(name, *shape, std=0.02, zeros=False, ones=False):
            if params is not None and name in params:
                return torch.as_tensor(params[name]).to(cfg.dtype)
            if ones:
                return torch.ones(*shape, dtype=cfg.dtype)
            if zeros:
                return torch.zeros(*shape, dtype=cfg.dtype)
            return rnd(*shape, std=std)

        dev = self.device
        r, tp = self.rank, self.tp
        self.alibi = None
        # The families share one transformer block; what differs is chosen here.  Every QKV projection is laid out
        # (K/V head, {its G query heads, k, v}, D), G = 1 outside Llama.
        llama = cfg.arch == "llama"
        self.G = nh // cfg.kv_heads
        self._split_qkv = self._split_rope if llama else self._split_rotary if cfg.rotary_dim else self._split
        self._mlp = self._mlp_swiglu if llama else self._mlp_act
        self._decode_attention = self._decode_attention_gqa if llama else self._decode_attention_mha
        # Llama's LM head runs the weight-streaming GEMV for 8 rows or fewer (a prefill's last tokens), the OPT
        # family's always the GEMM
        self.head_gemv = llama
        if llama:
            self._init_llama(params, rnd, fp8)
            return
        wte = get("embed_tokens", V, H)
        wte = F.pad(wte, (0, 0, 0, self.Vp - V))
        self.wte = wte[r * self.V_local:(r + 1) * self.V_local].contiguous().to(dev)     # vocab-parallel, tied head
        self.pos_offset = 2 if cfg.arch == "opt" else 0
        self.wpe = get("embed_positions", cfg.max_position_embeddings + self.pos_offset, H).to(dev) \
            if cfg.arch == "opt" else None

        def ln(name):                     # (gamma, beta, eps): what norm_rows and the decode GEMV's prologue take
            return get(name + ".g", H, ones=True).to(dev), get(name + ".b", H, zeros=True).to(dev), cfg.layer_norm_eps

        self.emb_ln = ln("emb_ln") if cfg.arch == "bloom" else None
        self.layers: List[Dict] = []
        hl = self.nh_local * self.D
        for i in range(cfg.num_hidden_layers):
            p = f"layers.{i}."
            qkv_w = get(p + "qkv.w", 3, nh, self.D, H)                  # [(q,k,v), head, D, H]
            # codegen has no attention biases (an all-zero bias is numerically the same and keeps one code path)
            qkv_b = get(p + "qkv.b", 3, nh, self.D, zeros=True)
            qkv_w, qkv_b = self._opt_qkv_rows(qkv_w), self._opt_qkv_rows(qkv_b)
            out_w = get(p + "out.w", H, H)[:, r * hl:(r + 1) * hl]
            fc1_w = get(p + "fc1.w", I, H)[r * (I // tp):(r + 1) * (I // tp)]
            fc1_b = get(p + "fc1.b", I, zeros=True)[r * (I // tp):(r + 1) * (I // tp)]
            fc2_w = get(p + "fc2.w", H, I)[:, r * (I // tp):(r + 1) * (I // tp)]
            self.layers.append({
                "ln1": ln(p + "ln1"),
                "ln2": ln(p + "ln2"),
                "qkv": _TPLinear(qkv_w.contiguous().to(dev), qkv_b.contiguous().to(dev), fp8),
                "out": _TPLinear(out_w.contiguous().to(dev), get(p + "out.b", H, zeros=True).to(dev) if r == 0 else None, fp8),
                "fc1": _TPLinear(fc1_w.contiguous().to(dev), fc1_b.contiguous().to(dev), fp8),
                "fc2": _TPLinear(fc2_w.contiguous().to(dev), get(p + "fc2.b", H, zeros=True).to(dev) if r == 0 else None, fp8),
            })
        self.final_ln = ln("final_ln")
        if cfg.tie_word_embeddings:
            self.head_w, self.head_b = self.wte, None
        else:                                                          # vocab-parallel like the embedding
            hw = F.pad(get("lm_head.w", V, H), (0, 0, 0, self.Vp - V))
            hb = F.pad(get("lm_head.b", V, zeros=True), (0, self.Vp - V))
            self.head_w = hw[r * self.V_local:(r + 1) * self.V_local].contiguous().to(dev)
            self.head_b = hb[r * self.V_local:(r + 1) * self.V_local].contiguous().to(dev)
        self.alibi = _alibi_slopes(nh)[r * self.nh_local:(r + 1) * self.nh_local].to(dev) if cfg.arch == "bloom" else None
        self._init_lora()

    def _opt_qkv_rows(self, w):
        """This rank's rows of the OPT-family QKV projection: w [(q, k, v), heads, D, ...] -> [(head, (q, k, v), D), ...]
        of its heads (a weight, a bias or a LoRA B)."""
        w = w[:, self.rank * self.nh_local:(self.rank + 1) * self.nh_local]
        return w.transpose(0, 1).reshape(3 * self.nh_local * self.D, *w.shape[3:])
    def _init_llama(self, params, rnd, fp8):
        """Weights of `GPTModel(arch="llama")` (its state_dict names and layouts), sliced for this rank: the QKV rows
        (K/V head, {G query heads, k, v}, D) and the interleaved (gate, up) rows of fc1 split by columns, the
        out-projection and fc2 by rows, the embedding and head by vocabulary."""
        cfg, dev, r, tp = self.cfg, self.device, self.rank, self.tp
        H, I, V, D, G = cfg.hidden_size, cfg.ffn_dim, cfg.vocab_size, self.D, self.G
        std = 0.02

        def get(name, *shape, ones=False):
            if params is not None:
                return torch.as_tensor(params[name]).to(cfg.dtype)
            return torch.ones(*shape, dtype=cfg.dtype) if ones else rnd(*shape, std=std)

        def rows(t, n):                   # this rank's n rows of a column-parallel weight
            return t[r * n:(r + 1) * n].contiguous().to(dev)

        wte = F.pad(get("wte", V, H), (0, 0, 0, self.Vp - V))
        self.wte = rows(wte, self.V_local)
        self.wpe, self.emb_ln, self.pos_offset = None, None, 0
        eps = cfg.layer_norm_eps
        self.layers = []
        qkv_local, hl, il = self.kv_local * (G + 2) * D, self.nh_local * D, I // tp
        for i in range(cfg.num_hidden_layers):
            p = f"blocks.{i}."
            self.layers.append({
                "ln1": ops.RMSNormArgs(get(p + "ln1_g", H, ones=True).to(dev), eps),
                "ln2": ops.RMSNormArgs(get(p + "ln2_g", H, ones=True).to(dev), eps),
                "qkv": _TPLinear(rows(get(p + "qkv_w", (G + 2) * cfg.kv_heads * D, H), qkv_local), None, fp8),
                "out": _TPLinear(get(p + "proj_w", H, H)[:, r * hl:(r + 1) * hl].contiguous().to(dev), None, fp8),
                "fc1": _TPLinear(rows(get(p + "fc1_w", 2 * I, H), 2 * il), None, fp8),
                "fc2": _TPLinear(get(p + "fc2_w", H, I)[:, r * il:(r + 1) * il].contiguous().to(dev), None, fp8),
            })
        self.final_ln = ops.RMSNormArgs(get("ln_f_g", H, ones=True).to(dev), eps)
        if cfg.tie_word_embeddings:
            self.head_w = self.wte
        else:
            self.head_w = rows(F.pad(get("decoder_w", V, H), (0, 0, 0, self.Vp - V)), self.V_local)
        self.head_b = None
        self._init_lora()

    # ------------------------------------------------------------------ LoRA adapters
    def _init_lora(self):
        """Stacked adapter tables, per layer and targeted projection: A [slots, R, K_local] and B [slots, N_local, R],
        zero in unused slots; fused projections stack their parts along R (each part rp rows: max_lora_rank rounded up
        to 8, ranks below it zero-padded), and B is block-diagonal over them."""
        cfg = self.cfg
        self.loras: Dict[str, Tuple[int, int]] = {}          # name -> (slot, load id)
        self.lora_slot_of: Dict[int, int] = {}               # load id -> slot
        self._lora_next_id = 1                               # load ids are never reused; 0 is the base model
        self._lora_pools = weakref.WeakSet()                 # pools whose prompts may use an adapter
        self.lora_rank_stride = rp = -(-cfg.max_lora_rank // 8) * 8
        if cfg.max_loras == 0 or cfg.arch not in LORA_TARGETS:
            return
        n, dt, dev = cfg.max_loras, cfg.dtype, self.device
        H, hl, il = cfg.hidden_size, self.nh_local * self.D, cfg.ffn_dim // self.tp
        # projection -> (N_local, K_local, stacked parts)
        shapes = {"qkv": (self.kv_local * (self.G + 2) * self.D, H, 3), "out": (H, hl, 1), "fc2": (H, il, 1)}
        if cfg.arch == "llama":
            shapes["fc1"] = (2 * il, H, 2)
        for l in self.layers:
            l["lora"] = {proj: (torch.zeros(n, k * rp, K, dtype=dt, device=dev),
                                torch.zeros(n, N, k * rp, dtype=dt, device=dev)) for proj, (N, K, k) in shapes.items()}
        self.lora_scale = torch.zeros(n, dtype=torch.float32, device=dev)

    def lora_id(self, name: str) -> int:
        """The load id of a loaded adapter (what `IterationLevelInputPool.enter_prompts(loras=...)` takes)."""
        if name not in self.loras:
            raise ValueError(f"unknown LoRA adapter {name!r}")
        return self.loras[name][1]

    def load_lora(self, name: str, tensors: Dict[str, torch.Tensor], alpha: float, r: int) -> int:
        """Copy an adapter into a free slot and return the slot.  `tensors`: PEFT names (`...layers.N.self_attn.q_proj.
        lora_A.weight` [r, in], `...lora_B.weight` [out, r]) of full, unsliced projections; a target it leaves out adds
        nothing.  The scale is alpha / r.  Raises ValueError when every slot is taken, r exceeds max_lora_rank, the
        architecture has no LoRA support (only Llama and OPT have) or a tensor is not a supported target of it."""
        cfg = self.cfg
        if cfg.arch not in LORA_TARGETS:
            raise ValueError(f"LoRA adapters are served for Llama and OPT models, not {cfg.arch!r}")
        if cfg.max_loras == 0:
            raise ValueError("this model has no LoRA slots (max_loras=0)")
        if name in self.loras:
            raise ValueError(f"LoRA adapter {name!r} is already loaded")
        if not 1 <= int(r) <= cfg.max_lora_rank:
            raise ValueError(f"LoRA rank {r} is outside 1..max_lora_rank={cfg.max_lora_rank}")
        used = set(s for s, _ in self.loras.values())
        free = [s for s in range(cfg.max_loras) if s not in used]
        if not free:
            raise ValueError(f"all {cfg.max_loras} LoRA slots are taken")
        tables = self._lora_tables(tensors, int(r))
        slot = free[0]
        for l, t in zip(self.layers, tables):
            for proj, (A, B) in t.items():
                l["lora"][proj][0][slot].copy_(A)
                l["lora"][proj][1][slot].copy_(B)
        self.lora_scale[slot] = float(alpha) / int(r)
        lid = self._lora_next_id
        self._lora_next_id += 1
        self.loras[name] = (slot, lid)
        self.lora_slot_of[lid] = slot
        return slot

    def unload_lora(self, name: str):
        """Free an adapter's slot.  Raises RuntimeError while a queued or running sequence uses it."""
        lid = self.lora_id(name)
        if any(pool.uses_lora(lid) for pool in list(self._lora_pools)):
            raise RuntimeError(f"LoRA adapter {name!r} is in use by a live sequence")
        slot, _ = self.loras.pop(name)
        del self.lora_slot_of[lid]
        for l in self.layers:
            for A, B in l["lora"].values():
                A[slot].zero_()
                B[slot].zero_()
        self.lora_scale[slot] = 0.0

    def _lora_tables(self, tensors, r: int):
        """Per layer, this rank's (A, B) of every projection in the slot layout (see `_init_lora`), built on the CPU."""
        cfg, rank, tp, rp = self.cfg, self.rank, self.tp, self.lora_rank_stride
        H, I, D = cfg.hidden_size, cfg.ffn_dim, self.D
        targets = LORA_TARGETS[cfg.arch]
        given: List[Dict[str, Dict[str, torch.Tensor]]] = [{} for _ in self.layers]
        for key, t in tensors.items():
            m = _LORA_NAME.search(key)
            if m is None:
                raise ValueError(f"not a LoRA tensor name: {key!r}")
            i, mod, ab = int(m.group(1)), m.group(2), m.group(3)
            if mod not in targets:
                raise ValueError(f"{mod!r} is not a supported LoRA target of {cfg.arch!r} (supported: "
                                 f"{sorted(targets)})")
            if not 0 <= i < len(self.layers):
                raise ValueError(f"LoRA tensor {key!r}: the model has {len(self.layers)} layers")
            given[i].setdefault(mod, {})[ab] = torch.as_tensor(t).float()
        llama = cfg.arch == "llama"
        dims = {"q_proj": (H, cfg.num_attention_heads * D), "k_proj": (H, cfg.kv_heads * D),
                "v_proj": (H, cfg.kv_heads * D), "o_proj": (H, H), "out_proj": (H, H), "gate_proj": (H, I),
                "up_proj": (H, I), "down_proj": (I, H), "fc2": (I, H)}
        hl, il = self.nh_local * D, I // tp
        out = []
        for i, g in enumerate(given):
            A, B = {}, {}                           # module -> A [rp, in], B [out, rp * parts] in its part's columns
            for mod, (proj, part) in targets.items():
                k_in, n_out = dims[mod]
                parts = 1 + max(p for pj, p in targets.values() if pj == proj)
                a, b = torch.zeros(rp, k_in), torch.zeros(n_out, parts * rp)
                if mod in g:
                    if set(g[mod]) != {"A", "B"}:
                        raise ValueError(f"layer {i} {mod}: needs both lora_A and lora_B")
                    ga, gb = g[mod]["A"], g[mod]["B"]
                    if tuple(ga.shape) != (r, k_in) or tuple(gb.shape) != (n_out, r):
                        raise ValueError(f"layer {i} {mod}: lora_A {tuple(ga.shape)} / lora_B {tuple(gb.shape)}, "
                                         f"expected {(r, k_in)} / {(n_out, r)}")
                    a[:r], b[:, part * rp:part * rp + r] = ga, gb
                A[mod], B[mod] = a, b
            t = {}
            if llama:
                qkv_local = self.kv_local * (self.G + 2) * D
                bq = pack_llama_qkv(B["q_proj"], B["k_proj"], B["v_proj"], cfg.kv_heads)
                t["qkv"] = (torch.cat([A["q_proj"], A["k_proj"], A["v_proj"]]),
                            bq[rank * qkv_local:(rank + 1) * qkv_local])
                bf = pack_llama_fc1(B["gate_proj"], B["up_proj"])
                t["fc1"] = (torch.cat([A["gate_proj"], A["up_proj"]]), bf[rank * 2 * il:(rank + 1) * 2 * il])
                o, d = "o_proj", "down_proj"
            else:
                nh = cfg.num_attention_heads
                b3 = torch.stack([B[m].view(nh, D, 3 * rp) for m in ("q_proj", "k_proj", "v_proj")])
                t["qkv"] = (torch.cat([A["q_proj"], A["k_proj"], A["v_proj"]]), self._opt_qkv_rows(b3))
                o, d = "out_proj", "fc2"
            # row-parallel layers: A sliced like the weight's columns, B whole
            t["out"] = (A[o][:, rank * hl:(rank + 1) * hl], B[o])
            t["fc2"] = (A[d][:, rank * il:(rank + 1) * il], B[d])
            out.append(t)
        return out

    # ------------------------------------------------------------------ cache
    def _new_kv(self, shape):
        if self.cfg.kv_cache_dtype == "fp8":
            return ops.Fp8KV.zeros(shape, self.device), ops.Fp8KV.zeros(shape, self.device)
        return (torch.zeros(shape, dtype=self.cfg.dtype, device=self.device),
                torch.zeros(shape, dtype=self.cfg.dtype, device=self.device))

    def init_cache(self, batch_size: int, max_len: int):
        """(reference: init_cache_np, opt_model.py:756) -> list of (k, v) [B, max_len, kv_heads_local, D]: bf16
        tensors, or ops.Fp8KV caches of that data shape when cfg.kv_cache_dtype is "fp8"."""
        return [self._new_kv((batch_size, max_len, self.kv_local, self.D)) for _ in self.layers]

    @staticmethod
    def _cache_write(kc, vc, k, v, at):
        """Write k / v [B, T, Hkv, D] into the cache: at rows at .. at + T - 1 of every sequence (`at` an int), or at
        the slots `at` (int64 [T], B = 1) of a slot-addressed cache."""
        slots = isinstance(at, torch.Tensor)
        if isinstance(kc, ops.Fp8KV):
            ops.fast.kv_cache_store(k, v, kc, vc, 0 if slots else at, at if slots else None)
        elif not slots:
            kc[:, at:at + k.shape[1]] = k
            vc[:, at:at + k.shape[1]] = v
        else:
            kc.index_copy_(0, at, k[0].contiguous())
            vc.index_copy_(0, at, v[0].contiguous())

    @staticmethod
    def _cache_read(kc, vc, end: int):
        """bf16 K / V [B, end, Hkv, D] of cache rows [0, end): views of a bf16 cache, a dequantised copy of an fp8 one."""
        if isinstance(kc, ops.Fp8KV):
            return ops.fast.kv_cache_load(kc, end), ops.fast.kv_cache_load(vc, end)
        return kc[:, :end], vc[:, :end]

    def weight_bytes(self) -> int:
        n = self.wte.numel() * 2 + (0 if self.head_w is self.wte else self.head_w.numel() * 2)
        for l in self.layers:
            n += sum(l[k].nbytes() for k in ("qkv", "out", "fc1", "fc2"))
        return n

    # ------------------------------------------------------------------ forward
    def _all_reduce(self, x, residual=None):
        """Sum over the tensor-parallel group (+ residual, fused into the one-shot kernel when it applies)."""
        if self.tp > 1:
            ar = self._nvls_allreduce(x, residual)
            if ar is not None:
                return ar
            dist.all_reduce(x, group=self.group)
        return x if residual is None else x + residual

    def _nvls_allreduce(self, x, residual=None):
        """In-switch (NVLS multimem) all-reduce of the activations through a symmetric buffer: two device-side
        barriers + one small kernel instead of an NCCL launch -- the latency that bounds tensor-parallel decode."""
        import os
        if self.__dict__.get("_nvls_state") == "off" or not x.is_cuda or x.dtype != torch.bfloat16 or \
                os.environ.get("ALPA_B200_SERVE_NVLS", "1") == "0":
            return None
        st = self.__dict__.get("_nvls_state")
        if st is None:
            try:
                from alpa_b200 import ops as _ops
                from alpa_b200.collective.fused import MultimemAllReduce
                if not _ops.native_available():
                    raise RuntimeError("native kernels unavailable")
                op = MultimemAllReduce(self.group, 16 << 20)           # 32 MiB of bf16
                if not op.available:
                    raise RuntimeError("no multicast mapping")
                st = self.__dict__["_nvls_state"] = op
            except Exception as e:  # noqa: BLE001
                import logging
                logging.getLogger(__name__).warning("NVLS all-reduce unavailable for serving (%s); using NCCL", e)
                self.__dict__["_nvls_state"] = "off"
                return None
        n = x.numel()
        n_pad = (n + 8 * self.tp - 1) // (8 * self.tp) * (8 * self.tp)
        if n_pad > st.numel:
            return None
        if n % 8 == 0 and n * 2 <= (256 << 10) and x.is_contiguous():
            # decode-sized message: ONE kernel (stage, barrier, in-switch reduce of the whole vector by every rank);
            # staging half and epoch are chosen on the device -> no per-call arguments, graph-replayable
            one = self.__dict__.get("_oneshot")
            if one is None:
                one = self.__dict__["_oneshot"] = {
                    "flags": _oneshot_flags(self.group), "counter": torch.zeros(1, dtype=torch.int32, device=x.device)}
            half = 1 << 20                                     # elements per staging half (2 MiB)
            res = None if residual is None else residual.contiguous()
            st.C.allreduce_oneshot(x, st.ws.ptrs[st.ws.rank], st.ws.multicast_ptr, half, x,
                                   one["flags"].peer_ptrs(0), one["counter"], st.ws.rank, res)
            return x
        buf = st.tensor[:n_pad]
        buf[:n].copy_(x.reshape(-1))
        if n_pad > n:
            buf[n:].zero_()
        st.ws.barrier()
        st.C.allreduce_multimem(st.ws.multicast_ptr, n_pad, st.ws.rank, st.tp, 8 if n_pad < (1 << 18) else 48)
        st.ws.barrier()
        x.copy_(buf[:n].view(x.shape))
        return x if residual is None else x + residual

    def _embed(self, input_ids, position_ids):
        x = ops.fast.embedding(input_ids, self.wte, self.rank * self.V_local)
        x = self._all_reduce(x)
        if self.wpe is not None:
            x = x + ops.fast.embedding(position_ids + self.pos_offset, self.wpe)
        if self.emb_ln is not None:
            x = ops.fast.norm_rows(x, self.emb_ln)
        return x

    # ---- the per-family pieces of the block, chosen in __init__
    def _split(self, qkv, position_ids):
        """q [B, T, kv_local, G, D], k / v [B, T, kv_local, D]: views of the projection qkv [B, T, kv_local, G + 2, D].
        No rotary."""
        G = self.G
        return qkv[:, :, :, :G], qkv[:, :, :, G], qkv[:, :, :, G + 1]

    def _split_rotary(self, qkv, position_ids):
        """`_split` with CodeGen's partial rotary (G = 1): the first rotary_dim channels of q and k rotated as
        interleaved pairs."""
        q, k, v = self._split(qkv, position_ids)
        rd = self.cfg.rotary_dim
        inv = 1.0 / (10000 ** (torch.arange(0, rd, 2, device=qkv.device, dtype=torch.float32) / rd))
        ang = position_ids[..., None].float() * inv            # [B, S, rd/2]
        sin, cos = ang.sin()[:, :, None, :], ang.cos()[:, :, None, :]

        def rot(t):
            t1, t2 = t[..., :rd:2].float(), t[..., 1:rd:2].float()
            out = torch.stack([t1 * cos - t2 * sin, t2 * cos + t1 * sin], dim=-1).flatten(-2)
            return torch.cat([out.to(t.dtype), t[..., rd:]], dim=-1)
        return rot(q[:, :, :, 0])[:, :, :, None], rot(k), v

    def _split_rope(self, qkv, position_ids):
        """`_split` with Llama's rotary: the query heads and k rotated in one kernel on the packed tensor."""
        return self._split(ops.fast.rotary_packed(qkv, position_ids, self.cfg.rope_theta, False), position_ids)

    def _mlp_act(self, l, h, ln=None, residual=None, lora=None):
        z = l["fc1"](h, self.cfg.activation, ln=ln)
        return self._lora(lora, l, "fc2", z, l["fc2"](z, residual=residual))

    def _mlp_swiglu(self, l, h, ln=None, residual=None, lora=None):
        gu = self._lora(lora, l, "fc1", h, l["fc1"](h, ln=ln))          # (gate, up) pairs interleaved
        z = ops.fast.swiglu(gu.view(*gu.shape[:-1], -1, 2))
        return self._lora(lora, l, "fc2", z, l["fc2"](z, residual=residual))

    def _lora(self, lora, l, proj, x, y):
        """y (the output of projection `proj` for input x, `ln` already applied) plus this rank's LoRA delta of the
        batch rows that carry an adapter, in place; `lora` = (rows, seg_start, seg_slot) or None (y unchanged)."""
        if lora is None:
            return y
        A, B = l["lora"][proj]
        x2, y2 = x.reshape(-1, x.shape[-1]), y.view(-1, y.shape[-1])
        ops.fast.lora_expand_(y2, ops.fast.lora_shrink(x2, A, *lora), B, self.lora_scale, *lora)
        return y

    def _decode_attention_mha(self, qkv, kc, vc, kv_len, position_ids, scale):
        q, k, v = self._split_qkv(qkv, position_ids)
        return ops.fast.decode_attention(q[:, :, :, 0], k, v, kc, vc, kv_len, scale)

    def _decode_attention_gqa(self, qkv, kc, vc, kv_len, position_ids, scale):
        return ops.fast.decode_attention_gqa(qkv, kc, vc, kv_len, position_ids, scale, self.cfg.rope_theta)

    def _head(self, x):
        """This rank's vocabulary shard of the logits of the last hidden states x [.., H]: final norm, LM head."""
        x = ops.fast.norm_rows(x.contiguous(), self.final_ln)
        if self.head_gemv and x.numel() // x.shape[-1] <= 8:
            return ops.fast.linear_decode(x, self.head_w, None)
        return ops.fast.linear(x, self.head_w, self.head_b)

    def _layers(self, x, position_ids, cache, attend, lora=None):
        """The transformer blocks over x [B, T, H].  `attend(q, k, v, kc, vc)` writes a layer's new K/V to its cache
        and returns the attention output of q [B, T, kv_local, G, D].  `lora` (see `forward_1d`) adds the adapters'
        deltas after every targeted projection, before the all-reduce of a row-parallel one."""
        B, T = x.shape[:2]
        for l, (kc, vc) in zip(self.layers, cache):
            h = ops.fast.norm_rows(x, l["ln1"])
            qkv = self._lora(lora, l, "qkv", h, l["qkv"](h))
            q, k, v = self._split_qkv(qkv.view(B, T, self.kv_local, self.G + 2, self.D), position_ids)
            o = attend(q, k, v, kc, vc).reshape(B, T, self.nh_local * self.D)
            a = self._lora(lora, l, "out", o, l["out"](o))
            if self.cfg.parallel_block:             # x + attn(ln(x)) + mlp(ln(x)): one all-reduce for both branches
                x = x + self._all_reduce(a + self._mlp(l, h))
                continue
            x = x + self._all_reduce(a)
            x = x + self._all_reduce(self._mlp(l, ops.fast.norm_rows(x, l["ln2"]), lora=lora))
        return x

    def forward(self, input_ids: torch.Tensor, position_ids: torch.Tensor, cache, cache_len: int,
                last_only: bool = True) -> torch.Tensor:
        """Run `input_ids` [B, T] whose first token sits at sequence position `cache_len`; appends K/V to the cache.
        Returns logits [B, 1 or T, V_local] (this rank's vocabulary shard)."""
        scale = 1.0 / math.sqrt(self.D)
        end = cache_len + input_ids.shape[1]

        def attend(q, k, v, kc, vc):
            self._cache_write(kc, vc, k, v, cache_len)
            kk, vv = self._cache_read(kc, vc, end)
            if self.alibi is not None:
                return self._attention_alibi(q[:, :, :, 0], kk, vv, scale, cache_len)
            # the grouped Q view against the valid cache rows: causal with Sq != Sk
            return ops.fast.attention(q, kk, vv, scale, True)[0]

        x = self._layers(self._embed(input_ids, position_ids), position_ids, cache, attend)
        return self._head(x[:, -1:] if last_only else x)

    def decode_step(self, input_ids: torch.Tensor, position_ids: torch.Tensor, cache, kv_len: torch.Tensor) -> torch.Tensor:
        """One new token per sequence with every position-dependent quantity on the device: `position_ids` [B, 1]
        (int64) is both the embedding position and the cache row to write, `kv_len` (int32 scalar tensor) the number
        of valid cache rows afterwards.  Shapes never change, so the step can be replayed from one CUDA graph.
        Returns logits [B, 1, V_local]."""
        assert self.alibi is None, "graph decode is implemented for learned / rotary position models"
        B = input_ids.shape[0]
        x = self._embed(input_ids, position_ids)
        scale = 1.0 / math.sqrt(self.D)
        for l, (kc, vc) in zip(self.layers, cache):
            # 5 launches per layer, 6 with Llama's SwiGLU (2 more under tensor parallelism): the norms ride in the GEMV
            # prologues, the cache append (and Llama's rotary) in the attention kernel, residual adds in the GEMV /
            # all-reduce epilogues
            qkv = l["qkv"](x, ln=l["ln1"]).view(B, 1, self.kv_local, self.G + 2, self.D)
            o = self._decode_attention(qkv, kc, vc, kv_len, position_ids, scale).reshape(B, 1, self.nh_local * self.D)
            if self.cfg.parallel_block:
                # both branches read LN1(x) (recomputed in the second GEMV's prologue); the MLP branch rides in as the
                # residual of the out-projection, the block input as the residual of the last GEMV / the all-reduce
                m = self._mlp(l, x, ln=l["ln1"], residual=x if self.tp == 1 else None)
                x = l["out"](o, residual=m) if self.tp == 1 else self._all_reduce(l["out"](o, residual=m), residual=x)
                continue
            if self.tp == 1:
                x = l["out"](o, residual=x)
                x = self._mlp(l, x, ln=l["ln2"], residual=x)
            else:
                x = self._all_reduce(l["out"](o), residual=x)
                x = self._all_reduce(self._mlp(l, x, ln=l["ln2"]), residual=x)
        # LM head: this rank's vocabulary shard of the weights streamed once per token, final norm in the prologue
        return ops.fast.linear_decode(x.contiguous(), self.head_w, None, self.head_b, ln=self.final_ln)

    # ------------------------------------------------------------------ ragged 1-D batches (iteration-level batching)
    def init_cache_1d(self, num_slots: int):
        """Slot-addressed cache: per layer (k, v) of [num_slots + 1, heads_local, D]; the last row is the scratch row
        padding tokens write to.  (reference: init_cache_np of opt_model_1d.py:457 -- a 1-D token cache)"""
        return [self._new_kv((num_slots + 1, self.kv_local, self.D)) for _ in self.layers]

    def forward_1d(self, input_ids: torch.Tensor, position: torch.Tensor, slot: torch.Tensor, seq_start: torch.Tensor,
                   ctx_len: torch.Tensor, cache, max_ctx: int, logit_index: torch.Tensor,
                   block_table: Optional[torch.Tensor] = None, block_size: Optional[int] = None,
                   chunks: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
                   n_prefill: int = 0,
                   lora: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
        """One iteration over a flat batch of T tokens that belong to different sequences (new prompts and running
        decodes mixed).  input_ids/position/slot: int64 [T]; seq_start/ctx_len: int32 [T] (see KVCacheManager.
        prepare_inputs).  K/V of every token go to cache row `slot`; attention reads each sequence's rows in place.
        A paged cache passes its int32 `block_table` and `block_size` (PagedKVCacheManager.prepare_inputs; seq_start
        is then a row of the table).  An empty `logit_index` (a batch of prefill chunks that end no prompt) still
        writes every token's K/V and returns no rows.
        `chunks` = (chunk_start, chunk_len, chunk_pos) int32 [P] of the batch's P prefill entries (prefix caching,
        PagedKVCacheManager.prepare_inputs) and `n_prefill` their total token count: those tokens, which come first,
        attend through `ops.paged_prefill_attention`, the decode and padding tokens after them through
        `ops.ragged_attention`.
        `lora` = (rows, seg_start, seg_slot) int32 (`ops.lora_shrink`): the batch rows that carry an adapter grouped
        by adapter slot; those rows get the adapter's delta after every targeted projection.  None = the base model.
        Returns logits [len(logit_index), V_local] of the rows in `logit_index` (the last token of every sequence).
        (reference: OPTForLMModule.__call__ of opt_model_1d.py:378 with fused_mmha)"""
        T = input_ids.shape[0]
        scale = 1.0 / math.sqrt(self.D)
        alibi = self.alibi.float().contiguous() if self.alibi is not None else None
        if chunks is not None and alibi is not None:
            raise ValueError("the paged prefill kernel takes no ALiBi")

        def attend(q, k, v, kc, vc):
            self._cache_write(kc, vc, k, v, slot)
            # the ragged kernel takes q as [T, heads, D] (a copy when G > 1), the prefill kernel reads the grouped view
            qh = q.reshape(T, self.nh_local, self.D)
            if chunks is None or n_prefill == 0:
                return ops.fast.ragged_attention(qh, kc, vc, seq_start, ctx_len, scale, max_ctx, alibi, block_table,
                                                 block_size)
            o = ops.fast.paged_prefill_attention(q[0, :n_prefill], kc, vc, block_table, block_size, *chunks, scale,
                                                 max_ctx)
            if n_prefill == T:
                return o
            r = ops.fast.ragged_attention(qh[n_prefill:], kc, vc, seq_start[n_prefill:], ctx_len[n_prefill:], scale,
                                          max_ctx, None, block_table, block_size)
            return torch.cat([o, r])

        # one batch row of T tokens
        x = self._layers(self._embed(input_ids.view(1, T), position.view(1, T)), position.view(1, T), cache, attend,
                         lora)
        if logit_index.numel() == 0:
            return x.new_empty(0, self.V_local)
        return self._head(x[0].index_select(0, logit_index))

    def _attention_alibi(self, q, k, v, scale, cache_len):
        B, T, h, D = q.shape
        S = k.shape[1]
        s = torch.einsum("bthd,bshd->bhts", q.float(), k.float()) * scale
        pos = torch.arange(S, device=q.device)
        s = s + self.alibi.view(1, h, 1, 1) * pos.view(1, 1, 1, S)
        qpos = cache_len + torch.arange(T, device=q.device)
        s = s.masked_fill(pos.view(1, 1, 1, S) > qpos.view(1, 1, T, 1), float("-inf"))
        p = torch.softmax(s, dim=-1)
        return torch.einsum("bhts,bshd->bthd", p, v.float()).to(q.dtype)

    def gather_logits(self, logits_local: torch.Tensor) -> torch.Tensor:
        """[.., V_local] per rank -> [.., V] (vocab-parallel LM head)."""
        if self.tp == 1:
            return logits_local[..., :self.cfg.vocab_size]
        parts = [torch.empty_like(logits_local) for _ in range(self.tp)]
        dist.all_gather(parts, logits_local.contiguous(), group=self.group)
        return torch.cat(parts, dim=-1)[..., :self.cfg.vocab_size]
