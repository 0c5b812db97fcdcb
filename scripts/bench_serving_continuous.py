"""Mixed-length serving workload: iteration-level batching (ragged 1-D batches) vs padded static batches.

Requests with prompt lengths and output lengths drawn from wide ranges arrive together; the metric is end-to-end
generated tokens/s and the mean / p90 request latency.  Static batching pads every batch to its longest prompt and
runs until its longest request finishes; the continuous engine retires requests individually.

    python scripts/bench_serving_continuous.py --model opt-125m --device cpu --requests 16      # smoke run on CPU
    python scripts/bench_serving_continuous.py --model opt-2.7b --weight-dtype fp8 --requests 256 (on an H100)

Paged against contiguous KV cache under one KV budget, where every request declares a cap above its true length:

    python scripts/bench_serving_continuous.py --model llama-3-8b --kv-block-size 0,16 --cache-tokens 32768 \
        --max-tokens 512 --min-new 16 --max-new 256

`--kv-block-size` alternates the modes (0 = contiguous) in one process on one model.  With `--max-tokens` each request
declares prompt + max_tokens as its length; its true output length is still drawn from [min_new, max_new], and the
sampler emits end-of-sequence there (the weights are random, so the model never would).  A contiguous cache reserves
the declared length, a paged one takes blocks as tokens arrive.

Prefix caching off against on, every request starting with the same 1024-token preamble:

    python scripts/bench_serving_continuous.py --model llama-3-8b --kv-block-size 16 --prefix-caching \
        --shared-prefix-tokens 1024 --requests 64 --min-prompt 16 --max-prompt 512

`--prefix-caching` runs every paged block size with caching off and on, alternated in one process; each run reports
its time to first token (p50 / p99, from the moment all requests are queued), the prompt tokens found in the cache
and the prompt tokens computed.

Multi-LoRA serving, the base model against 8 and 32 rank-16 adapters spread round robin over the requests:

    python scripts/bench_serving_continuous.py --model llama-3-8b --kv-block-size 16 --loras 0,8,32

`--loras` runs every mode once per adapter count, alternated in one process on one model (0 = no adapter).  The
adapters are random (every target of the architecture), so the outputs are meaningless and only the speed counts.
"""
import argparse
import json
import os
import random
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="opt-125m")
    p.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    p.add_argument("--weight-dtype", default="bf16", choices=["bf16", "fp8"])
    p.add_argument("--requests", type=int, default=64)
    p.add_argument("--min-prompt", type=int, default=16)
    p.add_argument("--max-prompt", type=int, default=512)
    p.add_argument("--min-new", type=int, default=8)
    p.add_argument("--max-new", type=int, default=128)
    p.add_argument("--batch-tokens", type=int, default=2048)
    p.add_argument("--static-batch", type=int, default=8)
    p.add_argument("--layers", type=int, default=None, help="override the layer count (smoke runs)")
    p.add_argument("--kv-cache-dtype", default="bf16", choices=["bf16", "fp8"])
    p.add_argument("--kv-block-size", default="0",
                   help="comma list of KV block sizes, run alternately; 0 = contiguous cache")
    p.add_argument("--cache-tokens", type=int, default=None,
                   help="KV cache size in tokens (default: every request's full length at once)")
    p.add_argument("--max-tokens", type=int, default=None,
                   help="the generation cap every request declares (default: its true output length)")
    p.add_argument("--prefix-caching", action="store_true",
                   help="run every paged block size with prefix caching off and on")
    p.add_argument("--shared-prefix-tokens", type=int, default=0,
                   help="every prompt starts with the same preamble of this many tokens")
    p.add_argument("--loras", default="0",
                   help="comma list of LoRA adapter counts spread over the requests, run alternately; 0 = base model")
    p.add_argument("--lora-rank", type=int, default=16)
    args = p.parse_args()
    from alpa_b200 import ops
    from alpa_b200.model.opt_model import DecoderLM, get_config
    from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator
    from alpa_b200.serve.generator import Generator
    dev = torch.device(args.device)
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    cfg = get_config(args.model, dtype=dtype, weight_dtype=args.weight_dtype, kv_cache_dtype=args.kv_cache_dtype)
    if args.layers:
        cfg.num_hidden_layers = args.layers
    lora_counts = [int(n) for n in args.loras.split(",")]
    cfg.max_loras, cfg.max_lora_rank = max(lora_counts), args.lora_rank
    model = DecoderLM(cfg, device=dev, seed=0)
    for i in range(cfg.max_loras):
        model.load_lora(f"a{i}", random_lora(cfg, args.lora_rank, seed=i), 2.0 * args.lora_rank, args.lora_rank)
    rnd = random.Random(0)
    preamble = [rnd.randint(4, cfg.vocab_size - 1) for _ in range(args.shared_prefix_tokens)]
    reqs = [(preamble + [rnd.randint(4, cfg.vocab_size - 1)
                         for _ in range(rnd.randint(args.min_prompt, args.max_prompt))],
             rnd.randint(args.min_new, args.max_new)) for _ in range(args.requests)]
    total_new = sum(n for _, n in reqs)

    def sync():
        if dev.type == "cuda":
            torch.cuda.synchronize()

    # ---- continuous batching
    per_seq = args.shared_prefix_tokens + args.max_prompt + max(args.max_new, args.max_tokens or 0) + 1
    cache_tokens = args.cache_tokens or min(per_seq * args.requests, 1 << 20)
    declared = [len(r[0]) + (args.max_tokens or r[1]) for r in reqs]
    eos = 2
    # a mode is (block size, prefix caching)
    # a mode is (block size, prefix caching, LoRA adapters)
    modes = [(int(b), c, n) for b in args.kv_block_size.split(",")
             for c in ((False, True) if args.prefix_caching and int(b) else (False,)) for n in lora_counts]
    engines = {}
    for bs, caching, n in modes:
        pc = InputPoolConfig(batch_size=args.batch_tokens, cache_size=cache_tokens, max_cache_per_seq=per_seq,
                             kv_block_size=bs or None, prefix_caching=caching)
        engines[(bs, caching, n)] = SequenceGenerator(model, pc)

    def run_continuous(mode):
        eng = engines[mode]
        pool = IterationLevelInputPool(eng.pool_config, pad_token_id=cfg.pad_token_id,
                                       eos_token_id=eos if args.max_tokens else -1, model=model)
        n = mode[2]
        loras = [model.lora_id(f"a{i % n}") if n else None for i in range(len(reqs))]
        ids = pool.enter_prompts([r[0] for r in reqs], max_lengths=declared, loras=loras)
        true_len = {sid: r[1] for sid, r in zip(ids, reqs)}
        stats = {"decode_iterations": 0, "decode_rows": 0, "ttft": {}}

        def stop_at_true_length(logits):
            rows = pool._current
            # decode rows: sequences that were decoding before this iteration (not a preempted sequence's re-prefill)
            decoding = sum(1 for p in rows if p.sentence_id in pool.wip)
            stats["decode_iterations"] += 1 if decoding else 0
            stats["decode_rows"] += decoding
            logits = logits.clone()
            logits[:, eos] = float("-inf")
            nxt = logits.argmax(-1)
            for r, p in enumerate(rows):
                if p.generation_length + 1 >= true_len[p.sentence_id]:
                    nxt[r] = eos
            return nxt
        sync()
        t0 = time.perf_counter()
        while not pool.is_finished():
            eng.step(pool, stop_at_true_length if args.max_tokens else None)
            if any(p.generation_length and p.sentence_id not in stats["ttft"]
                   for p in list(pool.wip.values()) + list(pool.done.values())):
                sync()
                now = time.perf_counter() - t0
                for p in list(pool.wip.values()) + list(pool.done.values()):
                    stats["ttft"].setdefault(p.sentence_id, now)
        sync()
        return time.perf_counter() - t0, pool.get_latency(), pool, stats

    results = {m: [] for m in modes}
    for m in modes:                                     # warm-up
        run_continuous(m)
    for _ in range(2 if len(modes) > 1 else 1):         # alternate the modes
        for m in modes:
            it0 = engines[m].iterations
            t, lat, pool, st = run_continuous(m)
            results[m].append((t, lat, engines[m].iterations - it0, pool, st))
    t_cont, lat_cont, iters, _, _ = min(results[modes[0]], key=lambda r: r[0])

    # ---- static padded batches (sorted by prompt length to be generous to the baseline)
    gen = Generator(model, args.static_batch, per_seq + 8)
    order = sorted(range(len(reqs)), key=lambda i: len(reqs[i][0]))

    def run_static():
        sync()
        t0 = time.perf_counter()
        lat = []
        for s in range(0, len(order), args.static_batch):
            grp = [reqs[i] for i in order[s:s + args.static_batch]]
            width = max(len(r[0]) for r in grp)
            ids = torch.tensor([[cfg.pad_token_id] * (width - len(r[0])) + r[0] for r in grp])
            gen.generate(ids, max_new_tokens=max(r[1] for r in grp))
            sync()
            lat += [time.perf_counter() - t0] * len(grp)
        return time.perf_counter() - t0, lat
    run_static()
    t_stat, lat_stat = run_static()

    def pct(xs, q):
        xs = sorted(xs)
        return xs[int(q * (len(xs) - 1))]
    print(json.dumps({
        "metric": f"{args.model} mixed-length serving throughput", "unit": "generated tokens/s",
        "continuous": {"tokens_per_s": total_new / t_cont, "seconds": t_cont, "iterations": iters,
                       "mean_latency_s": sum(lat_cont) / len(lat_cont), "p90_latency_s": pct(lat_cont, 0.9)},
        "static_padded": {"tokens_per_s": total_new / t_stat, "seconds": t_stat, "batch": args.static_batch,
                          "mean_latency_s": sum(lat_stat) / len(lat_stat), "p90_latency_s": pct(lat_stat, 0.9)},
        "speedup": t_stat / t_cont, "requests": args.requests, "generated_tokens": total_new,
        "kv_cache": [{"kv_block_size": bs or None, "prefix_caching": caching, "loras": n,
                      "tokens_per_s": total_new / t, "seconds": t, "iterations": it,
                      "tokens_per_s_runs": [total_new / r[0] for r in results[(bs, caching, n)]],
                      "mean_latency_s": sum(lat) / len(lat), "p90_latency_s": pct(lat, 0.9),
                      "mean_seqs_per_decode_iteration": st["decode_rows"] / max(1, st["decode_iterations"])
                      if args.max_tokens else None,
                      "preemptions": pool.num_preemptions, "peak_blocks": pool.peak_blocks_used if bs else None,
                      "ttft_p50_s": pct(list(st["ttft"].values()), 0.5),
                      "ttft_p99_s": pct(list(st["ttft"].values()), 0.99),
                      "prefix_hit_tokens": pool.prefix_hit_tokens if bs else None,
                      "prefill_tokens_computed": pool.prefill_tokens_computed if bs else None,
                      "cache_tokens": cache_tokens, "cache_bytes": ops.kv_cache_nbytes(engines[(bs, caching, n)].cache),
                      "kv_cache_dtype": args.kv_cache_dtype}
                     for bs, caching, n in modes
                     for t, lat, it, pool, st in [min(results[(bs, caching, n)], key=lambda r: r[0])]],
        "lora_rank": args.lora_rank if cfg.max_loras else None,
        "shared_prefix_tokens": args.shared_prefix_tokens,
        "declared_max_tokens": args.max_tokens,
        "prompt_len_range": [args.min_prompt, args.max_prompt], "new_tokens_range": [args.min_new, args.max_new],
        "weight_dtype": args.weight_dtype, "device": str(dev), "data": "synthetic prompts, random-init weights"}))


def random_lora(cfg, r, seed):
    """A random adapter on every LoRA target of cfg's architecture, under PEFT's tensor names."""
    from alpa_b200.model.opt_model import LORA_TARGETS
    H, I, D = cfg.hidden_size, cfg.ffn_dim, cfg.head_dim
    dims = {"q_proj": (H, cfg.num_attention_heads * D), "k_proj": (H, cfg.kv_heads * D),
            "v_proj": (H, cfg.kv_heads * D), "o_proj": (H, H), "out_proj": (H, H), "gate_proj": (H, I),
            "up_proj": (H, I), "down_proj": (I, H), "fc2": (I, H)}
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i in range(cfg.num_hidden_layers):
        for mod in LORA_TARGETS[cfg.arch]:
            k_in, n_out = dims[mod]
            out[f"layers.{i}.{mod}.lora_A.weight"] = torch.randn(r, k_in, generator=g) / k_in ** 0.5
            out[f"layers.{i}.{mod}.lora_B.weight"] = torch.randn(n_out, r, generator=g) * 0.01
    return out


if __name__ == "__main__":
    main()
