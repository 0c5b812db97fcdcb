"""OPT serving benchmark: p50 time-to-first-token and decode throughput (BASELINE.json config 5: OPT-2.7B, fp8, TP=8).

Launch: python scripts/bench_serving.py [--model opt-2.7b --prompt-len 512 --batch 1 --new-tokens 32 --weight-dtype fp8
        --kv-cache-dtype bf16]
        or under torchrun for tensor parallelism (one rank per GPU).  Synthetic prompts, random-init weights.
Metrics follow the reference's definitions (examples/llm_serving/generator.py:225-241): latency of the prompt phase,
tokens/s of generation."""
import argparse
import copy
import dataclasses
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--model", default="opt-2.7b")
    p.add_argument("--prompt-len", type=int, default=512)
    p.add_argument("--batch", type=int, default=1)
    p.add_argument("--new-tokens", type=int, default=32)
    p.add_argument("--trials", type=int, default=12)
    p.add_argument("--weight-dtype", default="fp8", choices=["bf16", "fp8"])
    p.add_argument("--kv-cache-dtype", default="bf16",
                   help="bf16 | fp8, or a comma list (e.g. bf16,fp8): one model, one generator per cache dtype, their "
                        "trials alternated in one session; one JSON line per cache dtype")
    p.add_argument("--profile", default="", help="write a per-kernel GPU time table of one generate() call here (diagnostic)")
    args = p.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    group = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
        group = dist.group.WORLD
    from alpa_b200 import ops
    from alpa_b200.model.opt_model import DecoderLM, get_config
    from alpa_b200.serve.generator import Generator
    kv_dtypes = args.kv_cache_dtype.split(",")
    cfg = get_config(args.model, weight_dtype=args.weight_dtype, kv_cache_dtype=kv_dtypes[0])
    model = DecoderLM(cfg, device="cuda", group=group, seed=0)
    gens = {}
    for d in kv_dtypes:
        # one shallow copy of the model per cache dtype: the weights are shared, each copy's cfg decides what its
        # init_cache allocates, and no model's cfg is changed after it was built
        m = model
        if d != cfg.kv_cache_dtype:
            m = copy.copy(model)
            m.cfg = dataclasses.replace(cfg, kv_cache_dtype=d)
        gens[d] = Generator(m, args.batch, args.prompt_len + args.new_tokens + 8)
    gen = gens[kv_dtypes[0]]
    g = torch.Generator().manual_seed(0)
    ttfts, decs = {d: [] for d in kv_dtypes}, {d: [] for d in kv_dtypes}
    for t in range(args.trials + 3):
        ids = torch.randint(4, cfg.vocab_size, (args.batch, args.prompt_len), generator=g)
        for d in kv_dtypes:
            if world > 1:
                dist.barrier()
            out = gens[d].generate(ids, max_new_tokens=args.new_tokens)
            v = torch.tensor([out.ttft_ms, out.decode_ms_per_token], device="cuda")
            if world > 1:
                dist.all_reduce(v, op=dist.ReduceOp.MAX)
            if t >= 3:
                ttfts[d].append(float(v[0]))
                decs[d].append(float(v[1]))
    if rank == 0:
        for d in kv_dtypes:
            print(json.dumps({"metric": f"{args.model} p50 TTFT", "value": statistics.median(ttfts[d]), "unit": "ms",
                              "p90_ttft_ms": sorted(ttfts[d])[int(0.9 * (len(ttfts[d]) - 1))],
                              "decode_ms_per_token_p50": statistics.median(decs[d]),
                              "decode_tokens_per_s": args.batch / (statistics.median(decs[d]) / 1e3),
                              "n_gpus": world, "weight_dtype": args.weight_dtype, "kv_cache_dtype": d,
                              "kv_cache_bytes_per_gpu": ops.kv_cache_nbytes(gens[d].cache),
                              "prompt_len": args.prompt_len, "batch": args.batch, "new_tokens": args.new_tokens,
                              "trials": args.trials, "weight_bytes_per_gpu": model.weight_bytes(),
                              "data": "synthetic prompts, random-init weights", "higher_is_better": False}))
    sys.stdout.flush()
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        ids = torch.randint(4, cfg.vocab_size, (args.batch, args.prompt_len), generator=g)
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            gen.generate(ids, max_new_tokens=args.new_tokens)
            torch.cuda.synchronize()
        if rank == 0:
            rows = {e.key: [e.count, e.device_time_total] for e in prof.key_averages()
                    if e.device_time_total > 0 and e.device_type.name == "CUDA"}
            os.makedirs(os.path.dirname(os.path.abspath(args.profile)), exist_ok=True)
            with open(args.profile, "w") as f:
                f.write(f"# GPU kernels of one generate() call: {args.model} {args.weight_dtype} prompt {args.prompt_len} "
                        f"+ {args.new_tokens} new tokens, {world} GPU(s); us total / calls / us per call\n")
                for name, (n, t) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
                    f.write(f"{t:10.1f} us {n:6d}x {t / n:8.2f} us  {name[:150]}\n")
    if world > 1:
        dist.barrier()
        os._exit(0)       # skip NCCL teardown: communicators referenced by captured graphs can block destroy


if __name__ == "__main__":
    main()
