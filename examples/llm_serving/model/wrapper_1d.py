"""Model factory for iteration-level (1-D) batching (reference: examples/llm_serving/model/wrapper_1d.py: InputPoolConfig,
SequenceGenerator, get_model(model_name, path, batch_size, cache_size)).

The engine itself is `alpa_b200.serve.batching.SequenceGenerator` (ragged 1-D token batches over a slot-addressed KV
cache, C++ cache manager, sm_90a ragged attention kernel); this module keeps the example-level entry point and the
return convention of the reference: `generate(...)` -> (output ids, per-sequence latency)."""
from __future__ import annotations

import os
from typing import List, Optional, Sequence

import numpy as np
import torch

from alpa_b200.model.opt_model import DecoderLM, get_config
from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator, pad, unpad  # noqa: F401
from alpa_b200.serve.generator import load_params_np


class WrappedSequenceGenerator:
    """`generate(input_ids, max_new_tokens=.., do_sample=..)` over padded arrays or ragged lists."""

    def __init__(self, engine: SequenceGenerator, model_name: str):
        self.engine, self.model_name = engine, model_name
        self.config = engine.model.cfg

    def _sampler(self, temperature: float, top_p: float):
        def sample(logits: torch.Tensor) -> torch.Tensor:
            probs = torch.softmax(logits.float() / max(temperature, 1e-6), dim=-1)
            if top_p < 1.0:
                sp, si = probs.sort(dim=-1, descending=True)
                sp = sp * ((sp.cumsum(-1) - sp) < max(top_p, 1e-6))
                return si.gather(-1, torch.multinomial(sp / sp.sum(-1, keepdim=True), 1))[:, 0]
            return torch.multinomial(probs, 1)[:, 0]
        return sample

    def generate(self, input_ids, max_length: Optional[int] = None, max_new_tokens: Optional[int] = None,
                 do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0, **unused):
        if max_length is None and max_new_tokens is None:
            raise RuntimeError("Please provide at least one of max_length and max_new_tokens.")
        if isinstance(input_ids, (np.ndarray, torch.Tensor)):
            input_ids = input_ids.tolist()
        prompts: List[List[int]] = unpad(input_ids, self.config.pad_token_id)
        eng, cfg = self.engine, self.config
        pool = IterationLevelInputPool(eng.pool_config, pad_token_id=cfg.pad_token_id, eos_token_id=2,
                                       max_length=max_length, max_new_tokens=max_new_tokens)
        pool.enter_prompts(prompts)
        sampler = self._sampler(temperature, top_p) if do_sample else None
        while not pool.is_finished():
            eng.step(pool, sampler)
        return pool.get_results(), pool.get_latency()


def get_model(model_name: str = "alpa/opt-1d-1.3b", path: Optional[str] = None, batch_size: int = 256,
              cache_size: int = 4096, max_cache_per_seq: int = 512, dummy: Optional[bool] = None,
              device: Optional[str] = None, weight_dtype: str = "bf16", group=None) -> WrappedSequenceGenerator:
    """`model_name`: "alpa/opt-1d-1.3b", "opt-1d-125m" or a plain architecture name ("opt-125m", "bloom-560m", ...).
    `batch_size`: tokens per iteration; `cache_size`: KV-cache slots (tokens) shared by all running sequences."""
    name = model_name.split("/", 1)[-1].replace("-1d-", "-")
    device = device or ("cuda" if torch.cuda.is_available() else "cpu")
    dtype = torch.bfloat16 if device == "cuda" else torch.float32
    cfg = get_config(name, dtype=dtype, weight_dtype=weight_dtype)
    params = None
    if path is not None and not dummy:
        params = load_params_np(cfg, os.path.join(os.path.expanduser(path), f"{name}_np"))
    model = DecoderLM(cfg, device=device, group=group, params=params)
    engine = SequenceGenerator(model, InputPoolConfig(batch_size=batch_size, cache_size=cache_size,
                                                      max_cache_per_seq=min(max_cache_per_seq, cache_size)))
    return WrappedSequenceGenerator(engine, model_name)
