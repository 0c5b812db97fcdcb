"""Iteration-level (continuous) batching: every model iteration runs a flat 1-D token batch that mixes newly admitted
prompts with one token of every running sequence, so a finished sequence frees its place immediately.

Reference: examples/llm_serving/model/opt_model_1d.py (PromptStatus:480, Prompt:486, IterationLevelInputPool:547 with
enter_prompts / next / update / get_results / get_latency, pad/unpad:716-738) and wrapper_1d.py (InputPoolConfig:28,
SequenceGenerator:34 generate / generate_by_batch).  The reference's cache bookkeeping lives in an external C++
package; here it is `alpa_b200._planner.KVCacheManager` (alpa_b200/csrc/serving_runtime.cpp) and the attention over
the ragged batch is `ops.ragged_attention` (sm_90a kernel).

With `InputPoolConfig(kv_block_size=...)` the cache is paged (`PagedKVCacheManager`): sequences take fixed-size blocks
as they grow instead of reserving their maximum length, a prompt longer than the token budget is prefilled in chunks,
and when the blocks run out the most recently admitted sequences are preempted and later recomputed.  With
`prefix_caching=True` as well, full blocks are shared between sequences whose token prefixes are equal: a new or
re-admitted prompt starts from the longest cached chain of blocks matching it and prefills only the rest, and that
suffix attends to the cached keys through `ops.paged_prefill_attention` (sm_90a kernel).

A prompt may name a LoRA adapter loaded into the model (`DecoderLM.load_lora`; `enter_prompts(loras=...)` takes its load
id).  `next()` then also lists the batch rows that carry an adapter, grouped by adapter slot, and the model adds each
adapter's delta to its rows (`ops.lora_shrink` / `ops.lora_expand_`).  With prefix caching, an adapter's blocks are
shared only between its own sequences (the load id is the block manager's namespace).
"""
from __future__ import annotations

import time
from collections import OrderedDict, deque
from dataclasses import dataclass
from enum import Enum
from typing import Deque, Dict, List, Optional, Sequence

import torch

from alpa_b200.model.opt_model import DecoderLM


class PromptStatus(Enum):
    PROMPT = 1
    DECODING = 2
    FINISHED = 3


class Prompt:
    """One sequence travelling through the pool."""

    def __init__(self, input_ids: Sequence[int], sentence_id: int, max_length: int = 2048, lora: Optional[int] = None):
        self.input_ids = list(input_ids)
        self.lora = lora                             # LoRA load id, None = the base model; kept across preemptions
        self.sentence_id = sentence_id
        self.max_length = max_length                 # prompt + generated, also the cache reservation
        self.status = PromptStatus.PROMPT
        self.generated_ids: List[int] = []
        self.start_time: Optional[float] = None
        self.finish_time: Optional[float] = None
        # paged cache: the tokens to prefill (the prompt, or prompt + generated after a preemption), how many of them
        # are in the cache, and the admission order preemption picks victims by
        self.fill_ids: List[int] = self.input_ids
        self.filled = 0
        self.admitted = 0

    @property
    def prompt_length(self) -> int:
        return len(self.input_ids)

    @property
    def generation_length(self) -> int:
        return len(self.generated_ids)

    @property
    def last_generated_id(self) -> int:
        return self.generated_ids[-1]

    def start(self):
        if self.start_time is None:               # a recomputed sequence keeps the start time of its first admission
            self.start_time = time.time()

    def add_token(self, token_id: int):
        self.generated_ids.append(int(token_id))
        self.status = PromptStatus.DECODING

    def finish(self, token_id: int):
        self.generated_ids.append(int(token_id))
        self.finish_time = time.time()
        self.status = PromptStatus.FINISHED

    @property
    def latency(self) -> float:
        if self.status != PromptStatus.FINISHED:
            raise RuntimeError("unfinished prompt")
        return self.finish_time - self.start_time


@dataclass
class InputPoolConfig:
    """batch_size = token budget of one iteration; cache_size = KV-cache slots (tokens) over all live sequences"""
    batch_size: int = 512
    cache_size: int = 4096
    max_cache_per_seq: int = 2048
    # an iteration's token count is padded up to a multiple of this (GEMM row alignment), not to the whole budget:
    # eager kernels need no fixed shapes, so a decode-only iteration of 12 sequences runs 16 rows, not `batch_size`
    # None = 8 on CPU, 128 on CUDA (one full GEMM row tile: decode is weight-bandwidth bound, so 128 rows cost what 16
    # do, and every kernel sees a shape it has been validated on)
    pad_multiple: Optional[int] = None
    # None = contiguous cache (every sequence reserves its maximum length); a power of two up to 1024 = paged cache of
    # cache_size / kv_block_size blocks taken on demand, with chunked prefill and recompute preemption
    kv_block_size: Optional[int] = None
    # share full blocks between sequences with equal token prefixes (needs kv_block_size >= 16, a bf16 cache and a
    # model without ALiBi); a prompt whose leading blocks are cached prefills only the rest
    prefix_caching: bool = False


class IterationLevelInputPool:
    """Admission + batch assembly.  `next()` returns the device-ready index arrays of one iteration, `update()` takes
    the sampled token of every sequence in that iteration."""

    def __init__(self, config: InputPoolConfig, pad_token_id: int = 1, eos_token_id: int = 2,
                 max_length: Optional[int] = None, max_new_tokens: Optional[int] = None,
                 model: Optional[DecoderLM] = None):
        """`model`: the model the pool's batches run on; prompts with a LoRA adapter need it (it maps load ids to
        slots and refuses to unload an adapter a queued or running prompt of this pool uses)."""
        from alpa_b200 import _planner
        self.config = config
        self.model = model
        if model is not None:
            model._lora_pools.add(self)
        self.batch_size = config.batch_size
        self.cache_size = config.cache_size
        self.max_length = max_length
        self.max_new_tokens = max_new_tokens
        self.pad, self.eos = pad_token_id, eos_token_id
        self.block_size = config.kv_block_size
        if self.block_size is None:
            self.cache_manager = _planner.KVCacheManager(config.cache_size)
        else:
            bs = self.block_size
            if not (isinstance(bs, int) and 1 <= bs <= 1024 and bs & (bs - 1) == 0):
                raise ValueError(f"kv_block_size must be a power of two up to 1024, got {bs!r}")
            if config.cache_size % bs:
                raise ValueError(f"cache_size {config.cache_size} is not a multiple of kv_block_size {bs}")
            if config.prefix_caching and bs < 16:
                raise ValueError(f"prefix_caching needs kv_block_size >= 16, got {bs}")
            self.cache_manager = _planner.PagedKVCacheManager(config.cache_size // bs, bs, config.prefix_caching)
        if config.prefix_caching and self.block_size is None:
            raise ValueError("prefix_caching needs a paged cache (kv_block_size)")
        self.prefix_caching = config.prefix_caching
        self.pad_slot = config.cache_size            # the scratch row of DecoderLM.init_cache_1d
        self.num_preemptions = 0
        self.peak_blocks_used = 0
        self.prefix_hit_tokens = 0                   # prompt tokens found in the cache, not computed
        self.prefill_tokens_computed = 0             # prompt (and recomputed) tokens run through the model
        self._admissions = 0
        self.todo: Deque[Prompt] = deque()
        self.wip: "OrderedDict[int, Prompt]" = OrderedDict()
        self.done: "OrderedDict[int, Prompt]" = OrderedDict()
        self._current: Optional[List[Prompt]] = None
        self._next_id = 1

    # ------------------------------------------------------------------ admission
    def is_finished(self) -> bool:
        return not self.todo and not self.wip

    def _reservation(self, prompt_len: int) -> int:
        n = self.config.max_cache_per_seq
        if self.max_length:
            n = min(n, self.max_length)
        if self.max_new_tokens:
            n = min(n, prompt_len + self.max_new_tokens)
        return max(n, prompt_len + 1)

    def accepts_prompt(self, prompt_len: int) -> bool:
        """Can this pool ever serve a prompt of `prompt_len` tokens?  It must leave room to generate within the
        per-sequence cap and the cache; a contiguous pool also prefills a prompt in one iteration."""
        cfg = self.config
        if prompt_len + 1 > min(cfg.max_cache_per_seq, cfg.cache_size):
            return False
        return self.block_size is not None or prompt_len <= cfg.batch_size

    def has_room_for(self, prompt_len: int, max_length: int) -> bool:
        """Would a new prompt still be admitted behind the queued ones in the next iteration?  Contiguous: its tokens
        fit the token budget and its `max_length` reservation fits the cache.  Paged: the queue is empty (a long
        prompt runs in chunks), or the queued prefill work plus this prompt fits the token budget and the free
        blocks."""
        if self.block_size is None:
            budget = self.batch_size - len(self.wip) - sum(p.prompt_length for p in self.todo)
            return prompt_len <= budget and self.cache_manager.can_allocate(
                [p.max_length for p in self.todo] + [max_length])
        if not self.todo:
            return True
        pending = [len(p.fill_ids) - p.filled for p in self.todo] + [prompt_len]
        blocks = sum(self.cache_manager.blocks_needed(p.sentence_id, len(p.fill_ids) - p.filled) for p in self.todo)
        blocks += -(-prompt_len // self.block_size) + len(self.wip)           # one block per decoder at most
        return sum(pending) <= self.batch_size - len(self.wip) and blocks <= self.cache_manager.num_free_blocks

    def enter_prompts(self, input_sequences: Sequence[Sequence[int]],
                      max_lengths: Optional[Sequence[int]] = None,
                      loras: Optional[Sequence[Optional[int]]] = None) -> List[int]:
        """Queue prompts; `max_lengths[i]` (prompt + generated) overrides the pool-wide limits for sequence i, and
        `loras[i]` is the load id (`DecoderLM.lora_id`) of its LoRA adapter, None for the base model."""
        ids = []
        paged = self.block_size is not None
        loras = [None] * len(input_sequences) if loras is None else list(loras)
        if len(loras) != len(input_sequences):
            raise ValueError("loras needs one entry per prompt")
        for lid in loras:
            if lid is not None and (self.model is None or lid not in self.model.lora_slot_of):
                raise ValueError(f"no LoRA adapter with load id {lid} is loaded in this pool's model")
        for i, seq in enumerate(input_sequences):
            if len(seq) == 0:
                raise ValueError("empty prompt")
            if len(seq) > self.batch_size and not paged:
                raise ValueError(f"prompt of {len(seq)} tokens exceeds the per-iteration token budget {self.batch_size}")
            cap = self.config.max_cache_per_seq
            if len(seq) >= cap:
                raise ValueError(f"prompt of {len(seq)} tokens leaves no room to generate within max_cache_per_seq={cap}")
            need = self._reservation(len(seq)) if max_lengths is None else max(int(max_lengths[i]), len(seq) + 1)
            # the attention kernel is launched with max_ctx = max_cache_per_seq: a longer reservation would make it
            # drop the newest keys silently, so the reservation is clamped (generation stops at the cap)
            need = min(need, cap)
            if paged:
                # nothing is reserved; a sequence may grow to the whole cache, never further (it could not be served)
                if len(seq) >= self.cache_size:
                    raise ValueError(f"prompt of {len(seq)} tokens leaves no room to generate in a cache of "
                                     f"{self.cache_size} tokens")
                need = min(need, self.cache_size)
            elif need > self.cache_size:
                raise ValueError(f"prompt needs {need} cache slots, the cache has {self.cache_size}")
            sid = self._next_id
            self._next_id += 1
            self.todo.append(Prompt(seq, sid, max_length=need, lora=loras[i]))
            ids.append(sid)
        return ids

    # ------------------------------------------------------------------ one iteration
    def next(self) -> Dict:
        """Admit as many queued prompts (FIFO) as the token budget and the cache allow, then lay the batch out:
        all tokens of each new prompt, one token per running sequence, padding."""
        if self.block_size is not None:
            return self._next_paged()
        decoding = list(self.wip.values())
        budget = self.batch_size - len(decoding)
        admitted: List[Prompt] = []
        used = 0
        while self.todo:
            p = self.todo[0]
            if used + p.prompt_length > budget:
                break
            if not self.cache_manager.can_allocate([q.max_length for q in admitted] + [p.max_length]):
                break
            admitted.append(self.todo.popleft())
            used += p.prompt_length
        for p in admitted:
            self.cache_manager.allocate(p.sentence_id, p.max_length)
            p.start()
        tokens = [t for p in admitted for t in p.input_ids] + [p.last_generated_id for p in decoding]
        width = self._width(len(tokens))
        idx = self.cache_manager.prepare_inputs([p.sentence_id for p in admitted], [p.prompt_length for p in admitted],
                                                [p.sentence_id for p in decoding], width, self.pad_slot)
        tokens = tokens + [self.pad] * (width - len(tokens))
        self._current = admitted + decoding
        lora = self._lora_segments([p.lora for p in admitted for _ in range(p.prompt_length)] +
                                   [p.lora for p in decoding])
        return {"input_ids": tokens, "num_new_prompts": len(admitted), "num_decoding": len(decoding), **idx, **lora}

    def _width(self, n_tokens: int) -> int:
        mult = max(1, self.config.pad_multiple or 8)
        width = min(self.batch_size, max(mult, (n_tokens + mult - 1) // mult * mult)) if mult > 1 else n_tokens
        return max(width, n_tokens)

    def _preempt(self, p: Prompt):
        """Return a running sequence's blocks and queue it at the front; it is recomputed from prompt + generated."""
        self.cache_manager.free(p.sentence_id)
        self.wip.pop(p.sentence_id, None)
        if p in self.todo:
            self.todo.remove(p)
        p.fill_ids = p.input_ids + p.generated_ids
        p.filled = 0
        p.status = PromptStatus.PROMPT
        self.todo.appendleft(p)
        self.num_preemptions += 1

    def _next_paged(self) -> Dict:
        """Paged iteration: secure one slot per decoding sequence (preempting the most recently admitted sequences
        while the blocks do not suffice), then admit prefill work FIFO while the token budget and the free blocks
        allow; a prefill that does not fit runs as a chunk and continues in the next iteration."""
        cm, bs = self.cache_manager, self.block_size
        preempted = False
        while True:
            decoding = list(self.wip.values())
            need = sum(cm.blocks_needed(p.sentence_id, 1) for p in decoding)
            if need <= cm.num_free_blocks:
                break
            holders = decoding + [p for p in self.todo if cm.has(p.sentence_id)]
            self._preempt(max(holders, key=lambda p: p.admitted))
            preempted = True
        free = cm.num_free_blocks - need
        budget = self.batch_size - len(decoding)
        chunks: List[tuple] = []                       # (prompt, tokens this iteration)
        # no prefill in an iteration that had to preempt: the freed blocks would be taken back at once
        for p in ([] if preempted else self.todo):
            if self.prefix_caching and budget > 0 and not cm.has(p.sentence_id):
                # admission (or re-admission after a preemption): start from the cached blocks of its prefix; cached
                # blocks it takes a reference on were counted as free
                before = cm.num_free_blocks
                hit = cm.match_prefix(p.sentence_id, p.fill_ids, p.lora or 0)
                free -= before - cm.num_free_blocks
                if free < 0:                           # the decoding sequences need those blocks: retry later
                    cm.free(p.sentence_id)
                    break
                p.filled = hit
                self.prefix_hit_tokens += hit
                self._admit(p)
            take = min(len(p.fill_ids) - p.filled, budget)
            room = free * bs
            if cm.has(p.sentence_id):                  # the unused rows of its last block
                room += -cm.length(p.sentence_id) % bs
            take = min(take, room)
            if take <= 0:
                break
            chunks.append((p, take))
            budget -= take
            free -= cm.blocks_needed(p.sentence_id, take)
            if p.filled + take < len(p.fill_ids):
                break
        ends = []
        for p, take in chunks:
            if not cm.has(p.sentence_id):
                cm.allocate(p.sentence_id, p.lora or 0)
                self._admit(p)
            ends.append(p.filled + take == len(p.fill_ids))
        tokens = [t for p, take in chunks for t in p.fill_ids[p.filled:p.filled + take]]
        tokens += [p.last_generated_id for p in decoding]
        width = self._width(len(tokens))
        mb = -(-self.config.max_cache_per_seq // bs)   # the kernel's table covers max_ctx = max_cache_per_seq keys
        # with prefix caching the manager learns every written position's token, so it can index the blocks filled
        ids = {"input_ids": tokens} if self.prefix_caching else {}
        idx = cm.prepare_inputs([p.sentence_id for p, _ in chunks], [take for _, take in chunks],
                                [p.sentence_id for p in decoding], width, self.pad_slot, ends, mb, **ids)
        for p, take in chunks:
            p.filled += take
            self.prefill_tokens_computed += take
        for p, end in zip([p for p, _ in chunks], ends):
            if end:
                self.todo.remove(p)
        self.peak_blocks_used = max(self.peak_blocks_used, cm.num_blocks - cm.num_free_blocks)
        tokens = tokens + [self.pad] * (width - len(tokens))
        self._current = [p for (p, _), end in zip(chunks, ends) if end] + decoding
        lora = self._lora_segments([p.lora for p, take in chunks for _ in range(take)] + [p.lora for p in decoding])
        return {"input_ids": tokens, "num_new_prompts": sum(ends), "num_decoding": len(decoding), **idx, **lora}

    def _lora_segments(self, row_loras: List[Optional[int]]) -> Dict:
        """`lora_rows` / `lora_seg_start` / `lora_seg_slot` (`ops.lora_shrink`) of the batch rows that carry an
        adapter, one segment per adapter in slot order; empty when no row does."""
        if all(lid is None for lid in row_loras):
            return {}
        by_slot: Dict[int, List[int]] = {}
        for row, lid in enumerate(row_loras):
            if lid is not None:
                by_slot.setdefault(self.model.lora_slot_of[lid], []).append(row)
        rows, starts, slots = [], [0], []
        for slot in sorted(by_slot):
            rows += by_slot[slot]
            starts.append(len(rows))
            slots.append(slot)
        return {"lora_rows": rows, "lora_seg_start": starts, "lora_seg_slot": slots}

    def uses_lora(self, load_id: int) -> bool:
        """Does a queued, running or just-batched prompt use this adapter?"""
        live = list(self.todo) + list(self.wip.values()) + list(self._current or [])
        return any(p.lora == load_id for p in live)

    def _admit(self, p: Prompt):
        self._admissions += 1
        p.admitted = self._admissions
        p.start()

    def _should_stop(self, p: Prompt, token: int) -> bool:
        if token == self.eos:
            return True
        n = p.generation_length + 1
        if self.max_new_tokens and n >= self.max_new_tokens:
            return True
        return p.prompt_length + n >= p.max_length

    def update(self, generated_ids: Sequence[int]):
        if self._current is None:
            raise RuntimeError("update() without a pending batch")
        assert len(generated_ids) >= len(self._current)
        for tok, p in zip(generated_ids, self._current):
            tok = int(tok)
            if self._should_stop(p, tok):
                self.wip.pop(p.sentence_id, None)
                p.finish(tok)
                self.cache_manager.free(p.sentence_id)
                self.done[p.sentence_id] = p
            else:
                p.add_token(tok)
                self.wip[p.sentence_id] = p
        self._current = None

    # ------------------------------------------------------------------ results
    def get_results(self) -> List[List[int]]:
        return [p.input_ids + p.generated_ids for _, p in sorted(self.done.items())]

    def get_latency(self) -> List[float]:
        return [p.latency for _, p in sorted(self.done.items())]

    def pop_finished(self) -> Dict[int, List[int]]:
        out = {sid: p.input_ids + p.generated_ids for sid, p in self.done.items()}
        self.done.clear()
        return out


def unpad(inputs, pad: int = 1) -> List[List[int]]:
    """Strip right padding (reference: unpad, opt_model_1d.py:716)"""
    if isinstance(inputs, torch.Tensor):
        inputs = inputs.tolist()
    out = []
    for seq in inputs:
        seq = list(seq)
        out.append(seq[:seq.index(pad)] if pad in seq else seq)
    return out


def pad(inputs, pad: int = 1) -> List[List[int]]:  # noqa: A001  (same name as the reference helper)
    if isinstance(inputs, torch.Tensor):
        inputs = inputs.tolist()
    n = max(len(s) for s in inputs)
    return [list(s) + [pad] * (n - len(s)) for s in inputs]


def check_prefix_caching(config: InputPoolConfig, model: DecoderLM):
    """Raise ValueError for a prefix-caching pool the model cannot serve: the suffix prefill runs on the paged
    prefill kernel, which takes a bf16 cache without ALiBi."""
    if not config.prefix_caching:
        return
    if config.kv_block_size is None or config.kv_block_size < 16:
        raise ValueError(f"prefix_caching needs kv_block_size >= 16, got {config.kv_block_size}")
    if model.alibi is not None:
        raise ValueError("prefix_caching is not supported with ALiBi models (BLOOM)")
    if model.cfg.kv_cache_dtype != "bf16":
        raise ValueError(f"prefix_caching is not supported with a {model.cfg.kv_cache_dtype} KV cache")


class SequenceGenerator:
    """Greedy generation with iteration-level batching over a DecoderLM (reference: wrapper_1d.SequenceGenerator:34)."""

    def __init__(self, model: DecoderLM, pool_config: Optional[InputPoolConfig] = None):
        self.model = model
        self.pool_config = pool_config or InputPoolConfig()
        check_prefix_caching(self.pool_config, model)
        if self.pool_config.pad_multiple is None:
            self.pool_config.pad_multiple = 128 if model.device.type == "cuda" else 8
        self.cache = model.init_cache_1d(self.pool_config.cache_size)
        self.iterations = 0
        self.tokens_processed = 0

    def _to_dev(self, batch: Dict):
        dev = self.model.device
        t = lambda x, dt: torch.tensor(x, dtype=dt, device=dev)  # noqa: E731
        return (t(batch["input_ids"], torch.long), t(batch["position"], torch.long), t(batch["slot"], torch.long),
                t(batch["seq_start"], torch.int32), t(batch["ctx_len"], torch.int32),
                t(batch["logit_index"], torch.long),
                t(batch["block_table"], torch.int32) if "block_table" in batch else None)

    def step(self, pool: IterationLevelInputPool, sampler=None) -> int:
        """Run one iteration for `pool`; returns the number of sequences that produced a token.  `sampler(logits
        [n, V]) -> ids [n]` replaces greedy argmax."""
        batch = pool.next()
        n = len(batch["logit_index"])
        if batch["num_tokens"] == 0:
            pool.update([])
            return 0
        ids, pos, slot, seq_start, ctx_len, logit_index, block_table = self._to_dev(batch)
        m = self.model
        paged = {} if block_table is None else {"block_table": block_table, "block_size": pool.block_size}
        if "lora_rows" in batch:
            paged["lora"] = tuple(torch.tensor(batch[k], dtype=torch.int32, device=m.device)
                                  for k in ("lora_rows", "lora_seg_start", "lora_seg_slot"))
        if "chunk_len" in batch and batch["chunk_len"]:
            dev = m.device
            paged["chunks"] = tuple(torch.tensor(batch[k], dtype=torch.int32, device=dev)
                                    for k in ("chunk_start", "chunk_len", "chunk_pos"))
            paged["n_prefill"] = sum(batch["chunk_len"])
        # a paged batch of prefill chunks that end no prompt has no logit rows, but its K/V must still be written
        logits = m.forward_1d(ids, pos, slot, seq_start, ctx_len, self.cache, pool.config.max_cache_per_seq, logit_index,
                              **paged)
        if n:
            logits = m.gather_logits(logits)
            nxt = logits.argmax(dim=-1) if sampler is None else sampler(logits)
            pool.update(nxt.tolist())
        else:
            pool.update([])
        self.iterations += 1
        self.tokens_processed += batch["num_tokens"]
        return n

    def generate(self, input_ids: Sequence[Sequence[int]], max_length: Optional[int] = None,
                 max_new_tokens: Optional[int] = None, loras: Optional[Sequence[Optional[str]]] = None,
                 **unused) -> List[List[int]]:
        """All prompts enter at once and drain through the iteration loop (reference: generate_by_batch).  `loras[i]`
        names the LoRA adapter of prompt i (`DecoderLM.load_lora`), None for the base model."""
        cfg = self.model.cfg
        ids = None if loras is None else [None if n is None else self.model.lora_id(n) for n in loras]
        pool = IterationLevelInputPool(self.pool_config, pad_token_id=cfg.pad_token_id, eos_token_id=2,
                                       max_length=max_length, max_new_tokens=max_new_tokens, model=self.model)
        pool.enter_prompts(input_ids, loras=ids)
        while not pool.is_finished():
            self.step(pool)
        self.last_latency = pool.get_latency()
        return pool.get_results()

    # the reference's name for the same loop (wrapper_1d.SequenceGenerator.generate_by_batch)
    generate_by_batch = generate
