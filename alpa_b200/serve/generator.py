"""Autoregressive generation on top of `alpa_b200.model.opt_model.DecoderLM`.

Reference: examples/llm_serving/generator.py (Generator:21 -- batches prompts, pads to buckets, calls the HF-style
`model.generate`), examples/llm_serving/model/wrapper.py (WrappedInferenceFunc / get_model:501 -- prompt processed in
chunks by the "encoder" executable, then one token per call of the "decoder" executable with the KV cache threaded
through), and the metric definitions in generator.py:225-241 (tokens/s, latency) that BASELINE.md cites.

TTFT (time to first token) = prompt forward + LM head + sampling of the first token, device-timed.
"""
from __future__ import annotations

import time
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Union

import torch

from alpa_b200.model.opt_model import DecoderLM, OPTConfig, get_config


@dataclass
class GenerationOutput:
    sequences: torch.Tensor                    # [B, prompt + new]
    ttft_ms: float = 0.0                       # device time of prefill + first sample
    decode_ms_per_token: float = 0.0
    num_new_tokens: int = 0
    logprobs: Optional[torch.Tensor] = None

    def tokens_per_second(self) -> float:
        total = self.ttft_ms + self.decode_ms_per_token * max(0, self.num_new_tokens - 1)
        return self.sequences.shape[0] * self.num_new_tokens / (total / 1e3) if total > 0 else 0.0


def _sample(logits: torch.Tensor, do_sample: bool, temperature: float, top_p: float, top_k: int,
            gen: Optional[torch.Generator]) -> torch.Tensor:
    """logits [B, V] (identical on every TP rank) -> token ids [B]"""
    if not do_sample:
        return logits.argmax(dim=-1)
    logits = logits.float() / max(temperature, 1e-5)
    if top_k and top_k > 0:
        kth = torch.topk(logits, min(top_k, logits.shape[-1]), dim=-1).values[..., -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    probs = torch.softmax(logits, dim=-1)
    if top_p < 1.0:
        sp, si = torch.sort(probs, dim=-1, descending=True)
        keep = (sp.cumsum(-1) - sp) < top_p
        sp = sp * keep
        probs = torch.zeros_like(probs).scatter_(-1, si, sp)
        probs = probs / probs.sum(-1, keepdim=True)
    return torch.multinomial(probs, 1, generator=gen).squeeze(-1)


class Generator:
    """HF-`generate`-style front end over a tensor-parallel DecoderLM (reference: get_model(...).generate)."""

    def __init__(self, model: DecoderLM, max_batch_size: int = 1, max_seq_len: int = 2048, seed: int = 0,
                 prefill_chunk: Optional[int] = None):
        self.model = model
        self.max_batch_size = max_batch_size
        self.max_seq_len = max_seq_len
        # prompts longer than `prefill_chunk` tokens enter the cache chunk by chunk (reference: the wrapper feeds long
        # prompts in fixed 64-token pieces against the preallocated cache, wrapper.py:243,450-478).  Bounds the
        # activation memory of the prompt phase; None = the whole prompt in one pass (flash attention needs no chunking)
        self.prefill_chunk = prefill_chunk
        self.cache = model.init_cache(max_batch_size, max_seq_len)
        self.rng = torch.Generator(device=model.device).manual_seed(seed)     # same seed -> same samples on all ranks
        # prompt phase replayed from a CUDA graph per (batch, prompt length): ~450 kernel launches collapse into one
        # graph launch, which is what bounds time-to-first-token for short prompts
        self.use_cuda_graph = model.device.type == "cuda"
        self._prefill_graphs: Dict = {}
        self._prefill_seen: Dict = {}
        self._decode_graphs: Dict = {}
        self._decode_seen: Dict = {}
        # static-shape decode replayed from one graph (device-side position / cache length); validated on hardware
        # (tests/test_zz_gpu_serving_1d.py); ALPA_B200_DECODE_GRAPH=0 turns it off
        import os as _os
        self.use_decode_graph = self.use_cuda_graph and _os.environ.get("ALPA_B200_DECODE_GRAPH", "1") != "0"

    # ---- front-end helpers of the reference's Generator (examples/llm_serving/generator.py)
    tokenizer = None          # anything with encode(str) -> ids / decode(ids) -> str; no tokenizer files are bundled

    @classmethod
    def load_model(cls, model_name: str, path: Optional[str] = None, tokenizer=None, **kwargs) -> "Generator":
        """Build the model and its generator (reference: Generator.load_model :88-131 -- tokenizer + model wrapper).
        `kwargs` go to `get_model` (batch_size, max_seq_len, dtype, weight_dtype, kv_cache_dtype, device, group)."""
        g = get_model(model_name, path=path, dummy=path is None, **kwargs)
        g.tokenizer = tokenizer
        return g

    def encode(self, text) -> list:
        """Token ids of a prompt: text needs `self.tokenizer`; lists of ids pass through (reference: encode :133-141)."""
        if isinstance(text, str):
            if self.tokenizer is None:
                raise ValueError("no tokenizer attached: pass token ids, or set `generator.tokenizer`")
            return [int(t) for t in self.tokenizer.encode(text)]
        return [int(t) for t in text]

    @torch.no_grad()
    def forward(self, input_ids: Union[torch.Tensor, Sequence[Sequence[int]]]) -> torch.Tensor:
        """Logits [B, T, V] of whole sequences in one pass (reference: Generator.forward :205-223, the scoring path of
        the logprobs endpoint).  Does not touch the generation cache."""
        m = self.model
        ids = input_ids if isinstance(input_ids, torch.Tensor) else torch.tensor([list(s) for s in input_ids])
        ids = ids.to(m.device)
        B, T = ids.shape
        cache = m.init_cache(B, T)
        pos = torch.arange(T, device=m.device).unsqueeze(0).expand(B, T)
        return m.gather_logits(m.forward(ids, pos, cache, 0, last_only=False))

    def estimate_performance(self, output_ids, latency: float, num_beams: int = 1, num_gpus: Optional[int] = None):
        """(TFLOPS per GPU, generated tokens / s, seconds per 32 tokens per sequence) of a finished batch
        (reference: estimate_performance :225-241; FLOPs = 2 x parameters-touched per token, attention included)."""
        cfg = self.model.cfg
        seqs = [list(s) for s in (output_ids.tolist() if isinstance(output_ids, torch.Tensor) else output_ids)]
        batch = num_beams * len(seqs)
        gen_len = max(len(s) for s in seqs)
        H, L, V = cfg.hidden_size, cfg.num_hidden_layers, cfg.vocab_size
        flops = batch * gen_len * (24 * H * H * L * (1 + gen_len / (6 * H)) + 2 * H * V)
        gpus = num_gpus or getattr(self.model, "tp", 1) or 1
        speed = batch * gen_len / latency
        return flops / latency / gpus / 1e12, speed, 32.0 / (speed / max(1, len(seqs)))

    def _decode(self, nxt: torch.Tensor, cache, B: int, cur: int) -> torch.Tensor:
        """Logits [B, V] of the token at sequence position `cur`.  On CUDA the whole step (~450 kernels) is one graph
        launch: token ids, position and cache length live in static device tensors that are updated in place."""
        m = self.model
        dev = m.device
        if not self.use_decode_graph or not self.use_cuda_graph or m.alibi is not None:
            p1 = torch.full((B, 1), cur, device=dev, dtype=torch.long)
            return m.gather_logits(m.forward(nxt[:, None], p1, cache, cur, last_only=True))[:, -1]
        entry = self._decode_graphs.get(B)
        if entry is None:
            st = self._decode_seen.setdefault(B, {"n": 0})
            if "ids" not in st:
                st["ids"] = torch.zeros(B, 1, dtype=torch.long, device=dev)
                st["pos"] = torch.zeros(B, 1, dtype=torch.long, device=dev)
                st["kv"] = torch.zeros(1, dtype=torch.int32, device=dev)
            st["ids"].copy_(nxt[:, None])
            st["pos"].fill_(cur)
            st["kv"].fill_(cur + 1)
            st["n"] += 1
            if st["n"] <= 2:                       # eager warm-up of the static-shape step
                return m.gather_logits(m.decode_step(st["ids"], st["pos"], cache, st["kv"]))[:, -1]
            try:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    out = m.gather_logits(m.decode_step(st["ids"], st["pos"], cache, st["kv"]))[:, -1]
                entry = (g, st, out)
                self._decode_graphs[B] = entry
                g.replay()
                return out.clone()
            except Exception as e:  # noqa: BLE001
                import logging
                logging.getLogger(__name__).warning("decode CUDA graph capture failed (%s); running eagerly", e)
                self.use_cuda_graph = False
                torch.cuda.synchronize()
                p1 = torch.full((B, 1), cur, device=dev, dtype=torch.long)
                return m.gather_logits(m.forward(nxt[:, None], p1, cache, cur, last_only=True))[:, -1]
        g, st, out = entry
        st["ids"].copy_(nxt[:, None])
        st["pos"].fill_(cur)
        st["kv"].fill_(cur + 1)
        g.replay()
        return out.clone()

    def _prefill(self, input_ids: torch.Tensor, pos: torch.Tensor, cache, B: int, T: int) -> torch.Tensor:
        m = self.model
        if self.prefill_chunk and T > self.prefill_chunk:
            logits = None
            for s0 in range(0, T, self.prefill_chunk):
                s1 = min(T, s0 + self.prefill_chunk)
                logits = m.gather_logits(m.forward(input_ids[:, s0:s1], pos[:, s0:s1], cache, s0, last_only=True))[:, -1]
            return logits
        if not self.use_cuda_graph:
            return m.gather_logits(m.forward(input_ids, pos, cache, 0, last_only=True))[:, -1]
        key = (B, T)
        entry = self._prefill_graphs.get(key)
        if entry is None:
            self._prefill_seen[key] = self._prefill_seen.get(key, 0) + 1
            if self._prefill_seen[key] < 2:          # first call of a shape: eager (allocator / NCCL warm-up)
                return m.gather_logits(m.forward(input_ids, pos, cache, 0, last_only=True))[:, -1]
            try:
                static_ids, static_pos = input_ids.clone(), pos.clone()
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    static_logits = m.gather_logits(m.forward(static_ids, static_pos, cache, 0, last_only=True))[:, -1]
                entry = (g, static_ids, static_pos, static_logits)
                self._prefill_graphs[key] = entry
            except Exception as e:  # noqa: BLE001
                import logging
                logging.getLogger(__name__).warning("prefill CUDA graph capture failed (%s); running eagerly", e)
                self.use_cuda_graph = False
                torch.cuda.synchronize()
                return m.gather_logits(m.forward(input_ids, pos, cache, 0, last_only=True))[:, -1]
        g, static_ids, static_pos, static_logits = entry
        static_ids.copy_(input_ids)
        static_pos.copy_(pos)
        g.replay()
        return static_logits.clone()

    @torch.no_grad()
    def generate(self, input_ids: Union[torch.Tensor, Sequence[Sequence[int]]], max_new_tokens: int = 32,
                 do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0, top_k: int = 0,
                 eos_token_id: Optional[int] = None, return_logprobs: bool = False, num_beams: int = 1,
                 length_penalty: float = 1.0) -> GenerationOutput:
        m = self.model
        dev = m.device
        if not isinstance(input_ids, torch.Tensor):
            if len({len(s) for s in input_ids}) > 1:
                # prompts of different lengths: no padding tokens enter the model -- the batch runs as a ragged 1-D
                # token batch (reference: wrapper.py pads and masks; opt_model_1d.py is its unpadded path)
                return self._generate_ragged(input_ids, max_new_tokens, do_sample, temperature, top_p, top_k,
                                             eos_token_id)
            input_ids = torch.tensor([list(s) for s in input_ids])
        input_ids = input_ids.to(dev)
        B, T = input_ids.shape
        if num_beams > 1:
            assert not do_sample, "beam search is deterministic (reference: launch_model_worker.py:64-67)"
            return self._beam_search(input_ids, max_new_tokens, num_beams, length_penalty, eos_token_id)
        assert B <= self.max_batch_size and T + max_new_tokens <= self.max_seq_len
        cache = [(k[:B], v[:B]) for k, v in self.cache]
        pos = torch.arange(T, device=dev).unsqueeze(0).expand(B, T)
        cuda = dev.type == "cuda"
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)] if cuda else None
        t0 = time.perf_counter()
        if cuda:
            ev[0].record()
        logits = self._prefill(input_ids, pos, cache, B, T)
        nxt = _sample(logits, do_sample, temperature, top_p, top_k, self.rng)
        if cuda:
            ev[1].record()
        t1 = time.perf_counter()
        out = [nxt]
        lps = [torch.log_softmax(logits.float(), -1).gather(-1, nxt[:, None])[:, 0]] if return_logprobs else None
        done = torch.zeros(B, dtype=torch.bool, device=dev)
        cur = T
        for _ in range(max_new_tokens - 1):
            if eos_token_id is not None:
                done |= nxt == eos_token_id
                if bool(done.all()):
                    break
            logits = self._decode(nxt, cache, B, cur)
            nxt = _sample(logits, do_sample, temperature, top_p, top_k, self.rng)
            if eos_token_id is not None:
                nxt = torch.where(done, torch.full_like(nxt, eos_token_id), nxt)
            out.append(nxt)
            if lps is not None:
                lps.append(torch.log_softmax(logits.float(), -1).gather(-1, nxt[:, None])[:, 0])
            cur += 1
        if cuda:
            ev[2].record()
            torch.cuda.synchronize()
            ttft, dec = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
        else:
            ttft, dec = (t1 - t0) * 1e3, (time.perf_counter() - t1) * 1e3
        n_new = len(out)
        seq = torch.cat([input_ids, torch.stack(out, dim=1)], dim=1)
        return GenerationOutput(seq, ttft, dec / max(1, n_new - 1), n_new,
                                torch.stack(lps, 1) if lps is not None else None)


    # ------------------------------------------------------------------ prompts of unequal length
    def _generate_ragged(self, prompts, max_new_tokens, do_sample, temperature, top_p, top_k, eos_token_id):
        from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator
        m = self.model
        longest = max(len(p) for p in prompts)
        assert len(prompts) <= self.max_batch_size and longest + max_new_tokens <= self.max_seq_len
        per_seq = longest + max_new_tokens
        mult = 128 if m.device.type == "cuda" else 8
        cfg = InputPoolConfig(batch_size=(max(sum(len(p) for p in prompts), len(prompts)) + mult - 1) // mult * mult,
                              cache_size=per_seq * len(prompts), max_cache_per_seq=per_seq)
        eng = self.__dict__.get("_ragged_engine")
        if eng is None or eng.pool_config.cache_size < cfg.cache_size:
            eng = self.__dict__["_ragged_engine"] = SequenceGenerator(m, cfg)
        cfg = InputPoolConfig(cfg.batch_size, eng.pool_config.cache_size, per_seq, eng.pool_config.pad_multiple)
        pool = IterationLevelInputPool(cfg, pad_token_id=m.cfg.pad_token_id,
                                       eos_token_id=-1 if eos_token_id is None else eos_token_id,
                                       max_new_tokens=max_new_tokens)
        pool.enter_prompts(prompts)
        t0 = time.perf_counter()
        sampler = (lambda lg: _sample(lg, do_sample, temperature, top_p, top_k, self.rng))
        first = None
        while not pool.is_finished():
            eng.step(pool, sampler)
            if first is None:
                first = time.perf_counter()
        total = time.perf_counter()
        res = pool.get_results()
        n_new = max(len(r) - len(p) for r, p in zip(res, prompts))
        width = max(len(r) for r in res)
        seq = torch.tensor([r + [m.cfg.pad_token_id] * (width - len(r)) for r in res], device=m.device)
        return GenerationOutput(seq, (first - t0) * 1e3, (total - first) * 1e3 / max(1, n_new - 1), n_new)

    # ------------------------------------------------------------------ beam search
    @staticmethod
    def reorder_cache(cache, beam_idx: torch.Tensor):
        """Row b of every cache tensor becomes old row beam_idx[b] (reference: the IndexSelect executable used to
        reorder the KV cache between beam-search steps, alpa/util.py:528-549, wrapper.py:115-182)."""
        for k, v in cache:
            k.copy_(k.index_select(0, beam_idx))
            v.copy_(v.index_select(0, beam_idx))

    def _beam_search(self, input_ids, max_new_tokens, num_beams, length_penalty, eos_token_id):
        """Standard beam search: `num_beams` live hypotheses per prompt, finished ones are ranked by
        sum-logprob / len**length_penalty.  Returns the best hypothesis per prompt (right-padded)."""
        m = self.model
        dev = m.device
        B, T = input_ids.shape
        nb = num_beams
        assert B * nb <= self.max_batch_size, "max_batch_size must cover batch * num_beams"
        assert T + max_new_tokens <= self.max_seq_len
        V = m.cfg.vocab_size
        ids = input_ids.repeat_interleave(nb, dim=0)                              # [B*nb, T]
        cache = [(k[:B * nb], v[:B * nb]) for k, v in self.cache]
        pos = torch.arange(T, device=dev).unsqueeze(0).expand(B * nb, T)
        t0 = time.perf_counter()
        logits = m.gather_logits(m.forward(ids, pos, cache, 0, last_only=True))[:, -1]
        score = torch.zeros(B, nb, device=dev)
        score[:, 1:] = float("-inf")                                              # identical beams: keep one at step 0
        seqs = torch.zeros(B * nb, 0, dtype=torch.long, device=dev)
        finished = [[] for _ in range(B)]                                         # (normalised score, tokens)
        cur = T
        t_first = None
        base = (torch.arange(B, device=dev) * nb)[:, None]
        for step in range(max_new_tokens):
            lp = torch.log_softmax(logits.float(), -1).view(B, nb, V) + score[:, :, None]
            top_s, top_i = lp.view(B, nb * V).topk(2 * nb, dim=-1)                # 2*nb candidates so that nb survive EOS
            src, tok = top_i // V, top_i % V
            new_score = torch.full((B, nb), float("-inf"), device=dev)
            new_src = torch.zeros(B, nb, dtype=torch.long, device=dev)
            new_tok = torch.zeros(B, nb, dtype=torch.long, device=dev)
            last = step == max_new_tokens - 1
            for b in range(B):
                n = 0
                for s_, src_, tok_ in zip(top_s[b].tolist(), src[b].tolist(), tok[b].tolist()):
                    if s_ == float("-inf"):
                        continue
                    hyp = seqs[b * nb + src_].tolist() + [tok_]
                    if (eos_token_id is not None and tok_ == eos_token_id) or last:
                        finished[b].append((s_ / (len(hyp) ** length_penalty), hyp))
                        if last:
                            n += 1
                            if n == nb:
                                break
                        continue
                    new_score[b, n], new_src[b, n], new_tok[b, n] = s_, src_, tok_
                    n += 1
                    if n == nb:
                        break
            if t_first is None:
                t_first = time.perf_counter()
            if last:
                break
            # stop early when no live hypothesis can beat the finished ones (scores only decrease)
            done = all(len(f) >= nb and max(x[0] for x in f) >= float(new_score[b].max()) / ((seqs.shape[1] + 1) ** length_penalty)
                       for b, f in enumerate(finished)) if eos_token_id is not None else False
            if done:
                break
            beam_idx = (base + new_src).view(-1)
            seqs = torch.cat([seqs.index_select(0, beam_idx), new_tok.view(-1, 1)], dim=1)
            self.reorder_cache(cache, beam_idx)
            score = new_score
            p1 = torch.full((B * nb, 1), cur, device=dev, dtype=torch.long)
            logits = m.gather_logits(m.forward(new_tok.view(-1, 1), p1, cache, cur, last_only=True))[:, -1]
            cur += 1
        t_end = time.perf_counter()
        best = [max(f, key=lambda x: x[0])[1] for f in finished]
        width = max(len(h) for h in best)
        pad = m.cfg.pad_token_id
        out = torch.tensor([h + [pad] * (width - len(h)) for h in best], device=dev)
        return GenerationOutput(torch.cat([input_ids, out], dim=1), (t_first - t0) * 1e3,
                                (t_end - t_first) * 1e3 / max(1, width - 1), width)


def get_model(model_name: str, path: Optional[str] = None, dummy: bool = True, batch_size: int = 1,
              max_seq_len: int = 2048, dtype=torch.bfloat16, weight_dtype: str = "bf16", device: str = "cuda",
              group=None, params: Optional[Dict] = None, kv_cache_dtype: str = "bf16") -> Generator:
    """HF-compatible entry (reference: get_model, wrapper.py:501).  `dummy=True` (or no `path`) uses random-init
    weights of the named architecture; `path` points to a directory of .npy weights in the reference's layout.
    `kv_cache_dtype="fp8"` keeps the KV cache in e4m3 with per-token, per-head scales (OPTConfig.kv_cache_dtype)."""
    cfg = get_config(model_name, dtype=dtype, weight_dtype=weight_dtype, kv_cache_dtype=kv_cache_dtype)
    if path is not None and not dummy:
        params = load_params_np(cfg, path)
    model = DecoderLM(cfg, device=device, group=group, params=params)
    return Generator(model, batch_size, max_seq_len)


def load_params_np(cfg: OPTConfig, path: str) -> Dict[str, torch.Tensor]:
    """Read per-tensor .npy files (reference: load_params_np, opt_model.py:875-1000 -- one file per parameter named
    `decoder.layers.N.self_attn.q_proj.weight` etc.) into the fused layout DecoderLM expects."""
    import os

    import numpy as np

    def ld(name):
        return torch.from_numpy(np.load(os.path.join(path, name)))
    H, nh, D = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim
    if cfg.arch == "bloom":
        return _load_bloom_params(cfg, ld)
    if cfg.arch == "codegen":
        return _load_codegen_params(cfg, ld)
    if cfg.arch == "llama":
        return _load_llama_params(cfg, path, ld)
    p: Dict[str, torch.Tensor] = {"embed_tokens": ld("decoder.embed_tokens.weight"),
                                  "embed_positions": ld("decoder.embed_positions.weight"),
                                  "final_ln.g": ld("decoder.layer_norm.weight"), "final_ln.b": ld("decoder.layer_norm.bias")}
    for i in range(cfg.num_hidden_layers):
        b = f"decoder.layers.{i}."
        q = [ld(b + f"self_attn.{n}_proj.weight").view(nh, D, H) for n in ("q", "k", "v")]
        qb = [ld(b + f"self_attn.{n}_proj.bias").view(nh, D) for n in ("q", "k", "v")]
        p[f"layers.{i}.qkv.w"] = torch.stack(q, 0)
        p[f"layers.{i}.qkv.b"] = torch.stack(qb, 0)
        p[f"layers.{i}.out.w"] = ld(b + "self_attn.out_proj.weight")
        p[f"layers.{i}.out.b"] = ld(b + "self_attn.out_proj.bias")
        p[f"layers.{i}.ln1.g"], p[f"layers.{i}.ln1.b"] = ld(b + "self_attn_layer_norm.weight"), ld(b + "self_attn_layer_norm.bias")
        p[f"layers.{i}.ln2.g"], p[f"layers.{i}.ln2.b"] = ld(b + "final_layer_norm.weight"), ld(b + "final_layer_norm.bias")
        p[f"layers.{i}.fc1.w"], p[f"layers.{i}.fc1.b"] = ld(b + "fc1.weight"), ld(b + "fc1.bias")
        p[f"layers.{i}.fc2.w"], p[f"layers.{i}.fc2.b"] = ld(b + "fc2.weight"), ld(b + "fc2.bias")
    return p


def load_lora_np(cfg: OPTConfig, path: str):
    """A PEFT LoRA adapter directory in the one-file-per-tensor form `load_params_np` reads: `adapter_config.json` (r,
    lora_alpha, target_modules) and one .npy file per tensor, named by PEFT (`base_model.model.model.layers.N.
    self_attn.q_proj.lora_A.weight`, with or without a .npy suffix).  Returns (tensors, alpha, r) for
    `DecoderLM.load_lora(name, *load_lora_np(cfg, path))`; raises ValueError for a target the model cannot serve."""
    import json
    import os

    import numpy as np

    from alpa_b200.model.opt_model import LORA_TARGETS
    with open(os.path.join(path, "adapter_config.json")) as f:
        conf = json.load(f)
    r, alpha = int(conf["r"]), float(conf.get("lora_alpha", conf["r"]))
    targets = LORA_TARGETS.get(cfg.arch)
    if targets is None:
        raise ValueError(f"LoRA adapters are served for Llama and OPT models, not {cfg.arch!r}")
    mods = conf.get("target_modules") or []
    mods = [mods] if isinstance(mods, str) else mods
    bad = sorted(set(mods) - set(targets))
    if bad:
        raise ValueError(f"unsupported LoRA target_modules {bad} for {cfg.arch!r} (supported: {sorted(targets)})")
    tensors = {}
    for name in os.listdir(path):
        if ".lora_A" in name or ".lora_B" in name:
            tensors[name.removesuffix(".npy")] = torch.from_numpy(np.load(os.path.join(path, name)))
    return tensors, alpha, r


def _load_bloom_params(cfg: OPTConfig, ld) -> Dict[str, torch.Tensor]:
    """Hugging Face BLOOM names (reference: load_params_np of bloom_model.py).  `query_key_value` rows are ordered
    [head, (q, k, v), D]."""
    H, nh, D = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim
    p = {"embed_tokens": ld("word_embeddings.weight"),
         "emb_ln.g": ld("word_embeddings_layernorm.weight"), "emb_ln.b": ld("word_embeddings_layernorm.bias"),
         "final_ln.g": ld("ln_f.weight"), "final_ln.b": ld("ln_f.bias")}
    for i in range(cfg.num_hidden_layers):
        b, o = f"h.{i}.", f"layers.{i}."
        p[o + "qkv.w"] = ld(b + "self_attention.query_key_value.weight").view(nh, 3, D, H).permute(1, 0, 2, 3).contiguous()
        p[o + "qkv.b"] = ld(b + "self_attention.query_key_value.bias").view(nh, 3, D).permute(1, 0, 2).contiguous()
        p[o + "out.w"], p[o + "out.b"] = ld(b + "self_attention.dense.weight"), ld(b + "self_attention.dense.bias")
        p[o + "ln1.g"], p[o + "ln1.b"] = ld(b + "input_layernorm.weight"), ld(b + "input_layernorm.bias")
        p[o + "ln2.g"], p[o + "ln2.b"] = ld(b + "post_attention_layernorm.weight"), ld(b + "post_attention_layernorm.bias")
        p[o + "fc1.w"], p[o + "fc1.b"] = ld(b + "mlp.dense_h_to_4h.weight"), ld(b + "mlp.dense_h_to_4h.bias")
        p[o + "fc2.w"], p[o + "fc2.b"] = ld(b + "mlp.dense_4h_to_h.weight"), ld(b + "mlp.dense_4h_to_h.bias")
    return p


def _load_llama_params(cfg: OPTConfig, path: str, ld) -> Dict[str, torch.Tensor]:
    """Hugging Face Llama names (`model.layers.N.self_attn.q_proj.weight`, ...; with or without the `model.` prefix)
    through `llama_params_from_hf` into the `GPTModel(arch="llama")` layout DecoderLM takes."""
    import os

    from alpa_b200.model.gpt_model import llama_params_from_hf
    from alpa_b200.model.opt_model import gpt_config_from_serving
    sd = {name: ld(name) for name in os.listdir(path) if name.endswith(".weight")}
    return llama_params_from_hf(sd, gpt_config_from_serving(cfg))


CODEGEN_MP_NUM = 4      # the released CodeGen checkpoints interleave qkv_proj for 4-way model parallelism


def _load_codegen_params(cfg: OPTConfig, ld) -> Dict[str, torch.Tensor]:
    """Hugging Face CodeGen names (reference: load_params_np of codegen_model.py:579-642).  `qkv_proj` rows are ordered
    [mp, (q, v, k), heads / mp, D]; there are no attention biases; the LM head is untied and has a bias."""
    H, nh, D = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim
    mp = CODEGEN_MP_NUM
    assert nh % mp == 0
    p = {"embed_tokens": ld("wte.weight"), "final_ln.g": ld("ln_f.weight"), "final_ln.b": ld("ln_f.bias"),
         "lm_head.w": ld("lm_head.weight"), "lm_head.b": ld("lm_head.bias")}
    for i in range(cfg.num_hidden_layers):
        b, o = f"h.{i}.", f"layers.{i}."
        w = ld(b + "attn.qkv_proj.weight").view(mp, 3, nh // mp, D, H)
        q, v, k = (w[:, j].reshape(nh, D, H) for j in range(3))
        p[o + "qkv.w"] = torch.stack([q, k, v], 0)
        p[o + "out.w"] = ld(b + "attn.out_proj.weight")
        p[o + "ln1.g"], p[o + "ln1.b"] = ld(b + "ln_1.weight"), ld(b + "ln_1.bias")
        p[o + "fc1.w"], p[o + "fc1.b"] = ld(b + "mlp.fc_in.weight"), ld(b + "mlp.fc_in.bias")
        p[o + "fc2.w"], p[o + "fc2.b"] = ld(b + "mlp.fc_out.weight"), ld(b + "mlp.fc_out.bias")
    return p


def pad_batch(inputs, pad_value, max_batch_size):
    """Right-pad every prompt to the longest one and the batch to `max_batch_size` rows, in place
    (reference: generator.pad_batch :244-260)."""
    max_len = max(len(x) for x in inputs)
    for x in inputs:
        x.extend([pad_value] * (max_len - len(x)))
    inputs.extend([[pad_value] * max_len for _ in range(max_batch_size - len(inputs))])
    return inputs


_serve_batch_counter = 0


def next_serve_batch_uuid(number: int = 1):
    """(reference: generator.next_serve_batch_uuid :265-273)"""
    global _serve_batch_counter
    first = _serve_batch_counter
    _serve_batch_counter += number
    return first if number == 1 else list(range(first, first + number))
