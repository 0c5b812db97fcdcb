"""Language-model worker: request queues with weighted fair sharing in front of the continuous-batching engine.

Reference: examples/llm_serving/launch_model_worker.py (LangModelWorker:36 -- `completions` / `logprobs` endpoints,
per-auth-group queues drained through NestedScheduler(WeightedRoundRobin) :90-112, a `batch_loop` :114 that forms
static batches of up to `max_bs` generate requests and serves logprob requests one at a time, request logging).

H100 design: the batch is not static.  The loop owns one `IterationLevelInputPool`; whenever the pool has token
budget and cache room left, the scheduler's next request is admitted, and every model iteration advances all running
sequences by one token, so short requests are not held back by long ones.  Logprob (scoring) requests run between
iterations on the padded path.
"""
from __future__ import annotations

import asyncio
import logging
import time
from collections import deque
from dataclasses import dataclass, field
from typing import Any, Dict, Hashable, List, Optional, Sequence

import torch

from alpa_b200.model.opt_model import DecoderLM
from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator
from alpa_b200.serve.scheduler import AsyncWrapper, FrontQueueScheduler, NestedScheduler, WeightedRoundRobin

logger = logging.getLogger(__name__)

DEFAULT_GROUP = "anonymous"
API_KEY_GROUP = "api_key"


@dataclass
class GenerateItem:
    uid: int
    prompt_ids: List[int]
    max_tokens: int
    future: asyncio.Future
    enqueue_time: float = field(default_factory=time.time)
    # sampling (temperature 0 = greedy), nucleus mass, no end-of-sequence before `min_tokens` generated tokens
    temperature: float = 0.0
    top_p: float = 1.0
    min_tokens: int = 0
    echo: bool = True
    lora: Optional[int] = None             # LoRA load id (DecoderLM.lora_id), None = the base model


@dataclass
class LogprobsItem:
    uid: int
    prompt_ids: List[int]
    top_k: int
    future: asyncio.Future
    enqueue_time: float = field(default_factory=time.time)
    lora: Optional[int] = None


class LangModelWorker:
    """`await worker.completions(ids, max_tokens)` / `await worker.logprobs(ids)`; `handle_request(request)` is the
    controller-facing entry ({"prompt_ids": [...], "max_tokens": n, "api_key": ...} or {"logprobs": true, ...})."""

    def __init__(self, model: DecoderLM, pool_config: Optional[InputPoolConfig] = None,
                 group_weights: Optional[Dict[Hashable, float]] = None,
                 api_key_weights: Optional[Dict[Hashable, float]] = None, default_api_key_weight: float = 1.0,
                 eos_token_id: int = 2, max_new_tokens_limit: int = 1024, tokenizer=None,
                 allowed_api_keys: Optional[Sequence[str]] = None, allow_non_key_access: bool = True,
                 max_seq_len_limit: Optional[int] = None):
        """`tokenizer`: anything with `encode(str) -> ids` / `decode(ids) -> str` (text prompts need one; pre-tokenised
        prompts do not).  `allowed_api_keys`: None = every key is accepted (keys only select the fair-share group);
        a list = requests with other keys are rejected.  `allow_non_key_access`: serve requests without a key.
        `max_seq_len_limit`: reject prompt + response lengths above it (reference: check_max_length_limit)."""
        self.tokenizer = tokenizer
        self.allowed_api_keys = None if allowed_api_keys is None else set(allowed_api_keys)
        self.allow_non_key_access = allow_non_key_access
        self.max_seq_len_limit = max_seq_len_limit
        self.model = model
        self.engine = SequenceGenerator(model, pool_config)
        self.pool = IterationLevelInputPool(self.engine.pool_config, pad_token_id=model.cfg.pad_token_id,
                                            eos_token_id=eos_token_id, model=model)
        self.max_new_tokens_limit = max_new_tokens_limit
        group_weights = dict(group_weights or {DEFAULT_GROUP: 1.0, API_KEY_GROUP: 4.0})
        inner = {g: deque() for g in group_weights}
        inner[API_KEY_GROUP] = WeightedRoundRobin(dict(api_key_weights or {}), 1.0, default_api_key_weight)
        group_weights.setdefault(API_KEY_GROUP, 4.0)
        self.request_queue = AsyncWrapper(FrontQueueScheduler(
            NestedScheduler(WeightedRoundRobin(group_weights, 1.0, None), inner)))
        self._uid = 0
        self._running: Dict[int, GenerateItem] = {}           # sentence id in the pool -> request
        self._task: Optional[asyncio.Task] = None
        self._wake: Optional[asyncio.Event] = None
        self.stats = {"completions": 0, "logprobs": 0, "iterations": 0, "generated_tokens": 0}

    # ------------------------------------------------------------------ public API
    def _enqueue(self, item, api_key: Optional[str]):
        if api_key is None:
            self.request_queue.put_nowait((DEFAULT_GROUP, item))
        else:
            self.request_queue.put_nowait((API_KEY_GROUP, (api_key, item)))
        self._ensure_loop()
        self._wake.set()

    async def completions(self, prompt_ids: Sequence[int], max_tokens: int = 16, api_key: Optional[str] = None,
                          temperature: float = 0.0, top_p: float = 1.0, min_tokens: int = 0, echo: bool = True,
                          lora: Optional[str] = None) -> Dict:
        """`temperature` 0 = greedy, > 0 = sample from softmax(logits / temperature) restricted to the smallest token
        set of mass `top_p`; no end-of-sequence before `min_tokens` new tokens; `echo` keeps the prompt in "ids";
        `lora` names a loaded LoRA adapter (ValueError for an unknown one), None = the base model."""
        lid = None if lora is None else self.model.lora_id(lora)
        if not (0.0 <= float(top_p) <= 1.0) or float(temperature) < 0.0:
            raise ValueError("need 0 <= top_p <= 1 and temperature >= 0")
        if len(prompt_ids) == 0:
            raise ValueError("empty prompt")
        if not self.pool.accepts_prompt(len(prompt_ids)):
            raise ValueError("prompt too long for this worker")
        max_tokens = max(1, min(int(max_tokens), self.max_new_tokens_limit))
        self._uid += 1
        fut = asyncio.get_running_loop().create_future()
        self._enqueue(GenerateItem(self._uid, list(map(int, prompt_ids)), max_tokens, fut,
                                   temperature=float(temperature), top_p=float(top_p),
                                   min_tokens=min(int(min_tokens), max_tokens - 1), echo=bool(echo), lora=lid), api_key)
        return await fut

    async def logprobs(self, prompt_ids: Sequence[int], top_k: int = 1, api_key: Optional[str] = None,
                       lora: Optional[str] = None) -> Dict:
        lid = None if lora is None else self.model.lora_id(lora)
        self._uid += 1
        fut = asyncio.get_running_loop().create_future()
        self._enqueue(LogprobsItem(self._uid, list(map(int, prompt_ids)), top_k, fut, lora=lid), api_key)
        return await fut

    # ---- request plumbing (reference: launch_model_worker.py normalize_prompts:231, check_max_length_limit:394,
    # get_authorization:403, get_remote_ip:429)
    def normalize_prompts(self, prompts) -> List[List[int]]:
        """A prompt is a string, a list of strings, a list of token ids or a list of lists of token ids: everything
        becomes the last form.  Text needs a tokenizer."""
        def enc(text: str) -> List[int]:
            if self.tokenizer is None:
                raise ValueError("this worker has no tokenizer: send pre-tokenised prompts (lists of token ids)")
            return [int(t) for t in self.tokenizer.encode(text)]
        try:
            if isinstance(prompts, str):
                prompts = [enc(prompts)]
            elif isinstance(prompts, (list, tuple)) and prompts and isinstance(prompts[0], str):
                assert all(isinstance(v, str) for v in prompts)
                prompts = [enc(p) for p in prompts]
            elif isinstance(prompts, (list, tuple)) and prompts and isinstance(prompts[0], int):
                prompts = [list(prompts)]
            assert isinstance(prompts, (list, tuple)) and len(prompts) > 0
            out = []
            for sub in prompts:
                assert isinstance(sub, (list, tuple)) and len(sub) > 0
                assert all(isinstance(v, int) and 0 <= v < self.model.cfg.vocab_size for v in sub)
                out.append([int(v) for v in sub])
            return out
        except AssertionError:
            raise ValueError("The prompt must be either a string, a list of strings, a list of integers, or a list of "
                             "integer lists (token ids inside the vocabulary).") from None

    def check_max_length_limit(self, cur_len: int, max_len: Optional[int] = None):
        max_len = max_len if max_len is not None else self.max_seq_len_limit
        if max_len is not None and cur_len > max_len:
            logger.info("Rejected a request with length = %d.", cur_len)
            raise ValueError(f"Your prompt length + response length = {cur_len} is too long: the limit is {max_len}.")

    def get_authorization(self, args: Dict, request=None) -> Optional[str]:
        """The fair-share key of a request: its api key when it is allowed, None for anonymous access."""
        api_key = args.get("api_key")
        if api_key is not None:
            if self.allowed_api_keys is not None and api_key not in self.allowed_api_keys:
                logger.error("Rejected a request with an incorrect key.")
                raise ValueError("API key is incorrect, please verify that you have passed the right value.")
            return api_key
        if not self.allow_non_key_access:
            logger.error("Rejected a request with no API key.")
            raise ValueError("This worker only serves requests that carry an API key.")
        return None

    @staticmethod
    def get_remote_ip(request) -> Optional[str]:
        scope = getattr(request, "scope", None) or {}
        for k, v in scope.get("headers", []):
            if k == b"x-forwarded-for":
                ip = v.decode().split(",")[0].strip()
                return ip[:ip.index(":")] if ":" in ip else ip
        client = getattr(request, "client", None)
        if client is not None:
            return getattr(client, "host", None) or (client[0] if isinstance(client, (tuple, list)) else None)
        return (scope.get("client") or [None])[0]

    async def handle_request(self, request) -> Dict:
        """{"prompt" | "prompt_ids": str | [str] | [int] | [[int]], "max_tokens": n, "api_key": ..., "logprobs": bool,
        "top_k": k, "lora": adapter name}.  One prompt -> the result dict; several prompts -> {"choices": [result, ...]} (served
        concurrently by the continuous-batching loop)."""
        obj = request.json() if hasattr(request, "json") else dict(request)
        api_key = self.get_authorization(obj, request)
        raw = obj.get("prompt_ids", obj.get("prompt"))
        if raw is None:
            raise ValueError('the request needs a "prompt" (text) or "prompt_ids" (token ids) field')
        prompts = self.normalize_prompts(raw)
        max_tokens = int(obj.get("max_tokens", 16))
        for p in prompts:
            self.check_max_length_limit(len(p) + (0 if obj.get("logprobs") else max_tokens))
        path = str(getattr(request, "path", "") or "").rstrip("/")
        want_logprobs = bool(obj.get("logprobs")) or path.endswith("/logprobs")
        if "stop" in obj:
            raise NotImplementedError("The stop argument is not implemented")
        lora = obj.get("lora")
        if lora is not None:
            self.model.lora_id(str(lora))                    # an unknown adapter fails the request before queueing
        if want_logprobs:
            coros = [self.logprobs(p, int(obj.get("top_k", 1)), api_key, lora) for p in prompts]
        else:
            # greedy unless the request asks for sampling (reference: temperature / top_p rounded to one decimal,
            # launch_model_worker.py:276-277)
            temperature = round(float(obj.get("temperature", 0.0)), 1)
            if obj.get("do_sample") and "temperature" not in obj:
                temperature = 1.0
            top_p = round(float(obj.get("top_p", 1.0)), 1)
            coros = [self.completions(p, max_tokens, api_key, temperature, top_p, int(obj.get("min_tokens", 0)),
                                      bool(obj.get("echo", True)), lora) for p in prompts]
        results = await asyncio.gather(*coros)
        if self.tokenizer is not None:
            for r in results:
                if isinstance(r, dict) and "ids" in r and "text" not in r:
                    r["text"] = self.tokenizer.decode(r["ids"])
        if path.endswith("/completions"):                    # OpenAI-style envelope (launch_model_worker.py:318-329)
            import uuid
            return {"id": str(uuid.uuid4()), "object": "text_completion", "created": int(time.time()),
                    "choices": list(results)}
        return results[0] if len(results) == 1 else {"choices": list(results)}

    async def shutdown(self):
        if self._task is not None:
            self._task.cancel()
            try:
                await self._task
            except asyncio.CancelledError:
                pass
            self._task = None

    # ------------------------------------------------------------------ the loop
    def _ensure_loop(self):
        if self._wake is None:
            self._wake = asyncio.Event()
        if self._task is None or self._task.done():
            self._task = asyncio.get_running_loop().create_task(self.batch_loop())

    @staticmethod
    def _unwrap(entry):
        group, payload = entry
        return payload[1] if group == API_KEY_GROUP else payload

    def _admit(self) -> Optional[LogprobsItem]:
        """Move requests from the scheduler into the pool while they fit; stop at the first logprob request (served
        by the caller) or the first generate request that has to wait (returned to the front of the queue)."""
        pool = self.pool
        while not self.request_queue.empty():
            entry = self.request_queue.get_nowait()
            item = self._unwrap(entry)
            if isinstance(item, LogprobsItem):
                return item
            need = max(min(len(item.prompt_ids) + item.max_tokens, pool.config.max_cache_per_seq, pool.cache_size),
                       len(item.prompt_ids) + 1)
            if not pool.has_room_for(len(item.prompt_ids), need):
                self.request_queue.put_nowait_special(lambda s, x: s.appendleft(x), entry)
                self.request_queue.task_done()            # the re-queued entry is counted again by put_nowait_special
                return None
            # stops after item.max_tokens tokens
            sid = pool.enter_prompts([item.prompt_ids], max_lengths=[need], loras=[item.lora])[0]
            self._running[sid] = item
        return None

    def _score(self, item: LogprobsItem) -> Dict:
        m = self.model
        ids = torch.tensor([item.prompt_ids], dtype=torch.long, device=m.device)
        T = ids.shape[1]
        pos = torch.arange(T, device=m.device)[None]
        if item.lora is None:
            logits = m.gather_logits(m.forward(ids, pos, m.init_cache(1, T), 0, last_only=False)).float()
        else:
            # adapters are served on the ragged path: the prompt as one sequence in a slot cache of its own
            i32 = lambda t: t.to(torch.int32)  # noqa: E731
            lora = (i32(pos[0]), torch.tensor([0, T], dtype=torch.int32, device=m.device),
                    torch.tensor([m.lora_slot_of[item.lora]], dtype=torch.int32, device=m.device))
            logits = m.gather_logits(m.forward_1d(ids[0], pos[0], pos[0], i32(pos[0] * 0), i32(pos[0] + 1),
                                                  m.init_cache_1d(T), T, pos[0], lora=lora))[None].float()
        lp_all = torch.log_softmax(logits[0], dim=-1)
        lp = lp_all[:-1]
        tok = lp.gather(-1, ids[0, 1:, None])[:, 0]
        k = max(1, item.top_k)
        top = lp.topk(k, dim=-1)
        nxt = lp_all[-1].topk(k)                       # the distribution after the last token (reference: logprobs
        return {"uid": item.uid, "token_logprobs": [None] + tok.tolist(), "top_ids": top.indices.tolist(),   # :332)
                "top_logprobs": top.values.tolist(), "next_ids": nxt.indices.tolist(),
                "next_logprobs": nxt.values.tolist()}

    def _needs_sampler(self) -> bool:
        return any(it.temperature > 0.0 or it.min_tokens > 0 for it in self._running.values())

    def _sample(self, logits: torch.Tensor) -> torch.Tensor:
        """Per-request next-token choice for the rows of the current iteration (`pool._current` gives the row
        order): greedy rows keep argmax; sampling rows draw from the temperature-scaled, top-p truncated
        distribution; rows still below their `min_tokens` cannot draw end-of-sequence."""
        rows = self.pool._current or []
        logits = logits[:len(rows)].float()
        eos = self.pool.eos
        for r, p in enumerate(rows):
            it = self._running.get(p.sentence_id)
            if it is not None and p.generation_length < it.min_tokens:
                logits[r, eos] = float("-inf")
        nxt = logits.argmax(dim=-1)
        for r, p in enumerate(rows):
            it = self._running.get(p.sentence_id)
            if it is None or it.temperature <= 0.0:
                continue
            probs = torch.softmax(logits[r] / it.temperature, dim=-1)
            if it.top_p < 1.0:
                sp, si = probs.sort(descending=True)
                keep = (sp.cumsum(0) - sp) < max(it.top_p, 1e-6)      # smallest prefix reaching top_p (>= 1 token)
                sp = sp * keep
                nxt[r] = si[torch.multinomial(sp / sp.sum(), 1)[0]]
            else:
                nxt[r] = torch.multinomial(probs, 1)[0]
        return nxt

    def _finish(self):
        for sid, seq in self.pool.pop_finished().items():
            item = self._running.pop(sid)
            n_new = len(seq) - len(item.prompt_ids)
            if not item.echo:
                seq = seq[len(item.prompt_ids):]
            self.stats["completions"] += 1
            self.stats["generated_tokens"] += n_new
            if not item.future.done():
                item.future.set_result({"uid": item.uid, "ids": seq, "num_new_tokens": n_new,
                                        "latency_s": time.time() - item.enqueue_time})
            self.request_queue.task_done()

    async def batch_loop(self):
        pool = self.pool
        while True:
            try:
                scoring = self._admit()
                if scoring is not None:
                    try:
                        scoring.future.set_result(self._score(scoring))
                    except Exception as e:  # noqa: BLE001
                        scoring.future.set_exception(e)
                    self.stats["logprobs"] += 1
                    self.request_queue.task_done()
                    continue
                if pool.is_finished():
                    self._wake.clear()
                    if self.request_queue.empty():
                        await self._wake.wait()
                    continue
                self.engine.step(pool, self._sample if self._needs_sampler() else None)
                self.stats["iterations"] += 1
                self._finish()
                await asyncio.sleep(0)                      # let new requests in between iterations
            except asyncio.CancelledError:
                raise
            except Exception as e:  # noqa: BLE001
                logger.exception("batch loop failed; failing the running requests")
                for item in self._running.values():
                    if not item.future.done():
                        item.future.set_exception(e)
                self._running.clear()
                self.pool = pool = IterationLevelInputPool(self.engine.pool_config, pad_token_id=self.model.cfg.pad_token_id,
                                                           eos_token_id=pool.eos, model=self.model)
