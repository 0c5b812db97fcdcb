"""Mixed-length serving workload: iteration-level batching (ragged 1-D batches) vs padded static batches.

Requests with prompt lengths and output lengths drawn from wide ranges arrive together; the metric is end-to-end
generated tokens/s and the mean / p90 request latency.  Static batching pads every batch to its longest prompt and
runs until its longest request finishes; the continuous engine retires requests individually.

    python scripts/bench_serving_continuous.py --model opt-125m --device cpu --requests 16      # smoke run on CPU
    python scripts/bench_serving_continuous.py --model opt-2.7b --weight-dtype fp8 --requests 256 (on an H100)
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
    args = p.parse_args()
    from alpa_b200.model.opt_model import DecoderLM, get_config
    from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator
    from alpa_b200.serve.generator import Generator
    dev = torch.device(args.device)
    dtype = torch.bfloat16 if dev.type == "cuda" else torch.float32
    cfg = get_config(args.model, dtype=dtype, weight_dtype=args.weight_dtype)
    if args.layers:
        cfg.num_hidden_layers = args.layers
    model = DecoderLM(cfg, device=dev, seed=0)
    rnd = random.Random(0)
    reqs = [([rnd.randint(4, cfg.vocab_size - 1) for _ in range(rnd.randint(args.min_prompt, args.max_prompt))],
             rnd.randint(args.min_new, args.max_new)) for _ in range(args.requests)]
    total_new = sum(n for _, n in reqs)

    def sync():
        if dev.type == "cuda":
            torch.cuda.synchronize()

    # ---- continuous batching
    per_seq = args.max_prompt + args.max_new + 1
    pc = InputPoolConfig(batch_size=args.batch_tokens, cache_size=min(per_seq * args.requests, 1 << 20),
                         max_cache_per_seq=per_seq)
    eng = SequenceGenerator(model, pc)

    def run_continuous():
        pool = IterationLevelInputPool(pc, pad_token_id=cfg.pad_token_id, eos_token_id=-1)
        pool.enter_prompts([r[0] for r in reqs], max_lengths=[len(r[0]) + r[1] for r in reqs])
        sync()
        t0 = time.perf_counter()
        while not pool.is_finished():
            eng.step(pool)
        sync()
        return time.perf_counter() - t0, pool.get_latency()
    run_continuous()                                    # warm-up
    it0 = eng.iterations
    t_cont, lat_cont = run_continuous()
    iters = eng.iterations - it0

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
        "prompt_len_range": [args.min_prompt, args.max_prompt], "new_tokens_range": [args.min_new, args.max_new],
        "weight_dtype": args.weight_dtype, "device": str(dev), "data": "synthetic prompts, random-init weights"}))


if __name__ == "__main__":
    main()
