#!/usr/bin/env python
"""Flagship benchmark: GPT training throughput through the public alpa_b200 API.

Reference benchmark: benchmark/alpa/benchmark_one_case_gpt_bert.py (GPT on synthetic all-ones-style
batches, AdamW with fp32 master weights, TFLOPs from alpa/util.py:1658-1687).  Config measured here
(BASELINE.json config 2): GPT-1.3B (S=1024, H=2048, L=24, heads=32, V=51200), bf16 compute, ShardParallel with the
auto-sharding ILP choosing the plan (`--method auto`, the default; the chosen logical mesh / plan is reported in the
JSON line), weak scaling (fixed per-GPU batch).  The step is replayed from a CUDA graph at every N; data-parallel
gradients live in static buckets reduced in-graph (in-switch NVLS multimem reduction, or bucketed NCCL).

    python bench.py --gpus N --steps K --warmup W          # N>1: launched under torchrun by the driver
    python bench.py --impl reference ...                    # the reference arm (unavailable offline)

Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time


def parse_args():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=8)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--impl", type=str, default="ours", choices=["ours", "reference", "torch"],
                   help="ours | reference (unmodified alpa, unavailable here) | torch (library baseline: cuBLAS + SDPA + "
                        "fused torch AdamW + DDP all-reduce, same model / batch / precision policy)")
    p.add_argument("--model", type=str, default="1.3B")
    p.add_argument("--batch-per-gpu", type=int, default=16)
    p.add_argument("--seq-len", type=int, default=1024)
    p.add_argument("--layers", type=int, default=None, help="debug only: override #layers (marks the run invalid)")
    p.add_argument("--method", type=str, default="auto", choices=["auto", "dp", "zero2", "zero3"],
                   help="auto = ShardParallel, the ILP picks the plan over every (d0, d1) logical mesh shape of the N GPUs; "
                        "dp / zero2 / zero3 force those plans")
    p.add_argument("--mesh-shape", type=str, default="auto", help="logical mesh for --method auto: 'auto' or e.g. 2x4")
    p.add_argument("--cuda-graph", type=int, default=int(os.environ.get("ALPA_B200_CUDA_GRAPH", "1")),
                   help="1 = replay the lowered step from a CUDA graph after two eager warm-up steps (default, every N)")
    p.add_argument("--nvls-allreduce", type=int, default=int(os.environ.get("ALPA_B200_NVLS_GRAD_ALLREDUCE", "-1")),
                   help="1 = gradient buckets reduced inside the NVSwitch (multimem.ld_reduce / multimem.st, device-side "
                        "barriers, captured in the graph); 0 = one NCCL all-reduce per bucket; -1 = auto (NVLS when N > 1)")
    p.add_argument("--nccl-max-ctas", type=int, default=8)
    p.add_argument("--grad-buckets", type=int, default=1, help="0 = one all-reduce per gradient (the round-1 behaviour)")
    p.add_argument("--profile", type=str, default="", help="write a per-kernel time table of one step here and exit")
    p.add_argument("--dump-outputs", type=str, default="",
                   help="after the timed steps, write what the last timed step returned (loss, a fixed seeded sample of "
                        "every updated parameter) as DIR/<name>.npy, float32, for output-for-output comparison of builds")
    return p.parse_args()


def torch_library_arm(args):
    """Library baseline of the same workload: plain PyTorch eager (cuBLAS GEMMs, library flash attention through SDPA,
    ATen LayerNorm/GELU/cross-entropy, torch.optim fused AdamW on fp32 master weights with bf16 autocast, DDP for
    N > 1).  This is the "NCCL + cuBLAS" comparison arm BASELINE.md asks for; none of alpa_b200's kernels run."""
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from alpa_b200.model.gpt_model import GPT_SPECS, GPTConfig, gpt_train_flops
    S_, H, L, heads, V = GPT_SPECS[args.model]
    if args.layers is not None:
        L = args.layers
    cfg = GPTConfig(vocab_size=V, hidden_size=H, num_hidden_layers=L, num_attention_heads=heads,
                    max_position_embeddings=S_)

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.qkv, self.proj = torch.nn.Linear(H, 3 * H), torch.nn.Linear(H, H)
            self.fc1, self.fc2 = torch.nn.Linear(H, 4 * H), torch.nn.Linear(4 * H, H)
            self.ln1, self.ln2 = torch.nn.LayerNorm(H, eps=1e-12), torch.nn.LayerNorm(H, eps=1e-12)

        def forward(self, x):
            B, S, _ = x.shape
            q, k, v = self.qkv(x).view(B, S, 3, heads, H // heads).permute(2, 0, 3, 1, 4)
            a = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, S, H)
            x = self.ln1(x + self.proj(a))
            return self.ln2(x + self.fc2(F.gelu(self.fc1(x))))

    class GPT(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.wte, self.wpe = torch.nn.Embedding(V, H), torch.nn.Embedding(S_, H)
            self.ln = torch.nn.LayerNorm(H, eps=1e-12)
            self.blocks = torch.nn.ModuleList([Block() for _ in range(L)])
            self.head = torch.nn.Linear(H, V)

        def forward(self, ids, pos):
            x = self.ln(self.wte(ids) + self.wpe(pos))
            for b in self.blocks:
                x = b(x)
            return self.head(x)

    torch.manual_seed(1234)
    model = GPT().cuda()
    ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank]) if world > 1 else model
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=1e-4, fused=True)
    B, S = args.batch_per_gpu, args.seq_len
    g = torch.Generator().manual_seed(7 + rank)
    host = {"ids": torch.randint(1, V, (B, S), generator=g).pin_memory(), "pos": torch.arange(S).repeat(B, 1).pin_memory(),
            "labels": torch.randint(1, V, (B, S), generator=g).pin_memory()}

    def step(batch):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = ddp(batch["ids"], batch["pos"])
        loss = F.cross_entropy(logits.float().view(-1, V), batch["labels"].view(-1))
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss

    dev = {k: v.cuda() for k, v in host.items()}
    for _ in range(max(3, args.warmup)):
        step(dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
    sampler = ClockSampler(local_rank)
    sampler.start()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = step(dev)
    e1.record()
    barrier()
    dev_ms = e0.elapsed_time(e1) / args.steps
    barrier()
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    for _ in range(args.steps):
        loss = step({k: v.cuda(non_blocking=True) for k, v in host.items()})
        _ = float(loss)
    f1.record()
    barrier()
    e2e_ms = f0.elapsed_time(f1) / args.steps
    sampler.stop_flag.set()
    sampler.join(timeout=2)
    t = torch.tensor([dev_ms, e2e_ms], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, e2e_ms = float(t[0]), float(t[1])
    tokens = B * S * world
    tflops = gpt_train_flops(B * world, S, cfg) / (dev_ms / 1e3) / world / 1e12
    if rank == 0:
        print(json.dumps({
            "metric": "GPT-1.3B training throughput (tokens/s, whole job); PFLOPS-util in extra fields",
            "value": tokens / (dev_ms / 1e3), "unit": "tokens/s", "n_gpus": world, "steps": args.steps,
            "warmup": max(3, args.warmup), "ms_per_step": dev_ms, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": tflops / 37.01, "dtype": "bf16 autocast, fp32 master", "data": "synthetic random tokens, random-init weights",
            "impl": "torch-library-baseline (cuBLAS + SDPA + fused torch AdamW + DDP)", "tflops_per_gpu": tflops,
            "e2e": {"value": tokens / (e2e_ms / 1e3), "unit": "tokens/s", "ms_per_step": e2e_ms,
                    "h2d_bytes_per_step": sum(v.numel() * v.element_size() for v in host.values()), "d2h_bytes_per_step": 4},
            "gpu_launches": 0, "clocks": sampler.summary(),
            "config": {"model": f"GPT-{args.model}", "global_batch": B * world, "seq_len": S, "parallelism": f"ddp{world}"}}),
            flush=True)
    if world > 1:
        dist.barrier()
        os._exit(0)
    return 0


def reference_arm(args):
    """The unmodified reference (alpa, looked up under baseline/_ref) needs jax 0.3.22 + flax + ray + the
    jaxlib-alpa XLA fork (bazel build); it is reported as unavailable when it cannot be imported."""
    why = "reference needs jax==0.3.22, flax, ray and the jaxlib-alpa XLA fork (bazel build); not in the offline wheelhouse"
    try:
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "baseline", "_ref"))
        import alpa  # noqa: F401
        why = "reference imported but its jaxlib-alpa XLA backend is not installed"
    except Exception as e:  # noqa: BLE001
        why = f"import alpa failed: {type(e).__name__}: {str(e)[:120]} ({why})"
    print(json.dumps({"impl": "reference", "unavailable": why}))
    return 0


class ClockSampler(threading.Thread):
    """Samples SM clocks / throttle reasons with nvidia-smi while the timed region runs."""

    def __init__(self, gpu_index: int):
        super().__init__(daemon=True)
        self.gpu = gpu_index
        self.samples = []
        self.stop_flag = threading.Event()

    def run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        while not self.stop_flag.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                                      str(self.gpu)], capture_output=True, text=True, timeout=5).stdout.strip()
                parts = [x.strip() for x in out.split(",")]
                if len(parts) >= 7:
                    self.samples.append(parts)
            except Exception:  # noqa: BLE001
                pass
            self.stop_flag.wait(0.2)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        sm = sorted(float(s[0]) for s in self.samples if s[0].replace(".", "").isdigit())
        mx = [float(s[1]) for s in self.samples if s[1].replace(".", "").isdigit()]
        reasons = set()
        for s in self.samples:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), s[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(self.samples)}


DUMP_BUDGET = 16 * 1024 * 1024   # float32 elements in all (64 MB); shared out evenly over the parameters


def dump_outputs(out_dir, loss, state):
    """Loss and updated parameters of the last timed step as float32 .npy files (the inputs are seeded, so two builds
    of the project can be compared output for output).  A parameter larger than its share of the 64 MB budget is
    represented by a fixed seeded sample of its elements.  Written by rank 0 from the values it holds: with a sharded
    plan (--method zero3 or a tensor-parallel mesh) that is rank 0's shard of each parameter."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)

    def host(x):
        x = getattr(x, "_value", x)
        return x.detach().float().cpu() if isinstance(x, torch.Tensor) else torch.as_tensor(x, dtype=torch.float32)
    np.save(os.path.join(out_dir, "loss.npy"), host(loss).numpy().reshape(-1))
    params = sorted(state.params.items())
    per_param = max(1, (DUMP_BUDGET - 1) // max(1, len(params)))
    for name, p in params:
        flat = host(p).reshape(-1)
        if flat.numel() > per_param:
            g = torch.Generator().manual_seed(0)
            idx = torch.randint(0, flat.numel(), (per_param,), generator=g).sort().values
            flat = flat[idx]
        np.save(os.path.join(out_dir, f"param.{name}.npy"), flat.numpy())


def main():
    args = parse_args()
    if args.impl == "reference":
        return reference_arm(args)
    if args.impl == "torch":
        return torch_library_arm(args)

    import torch
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and world > 1:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}")
    os.environ.setdefault("ALPA_B200_REQUIRE_NATIVE", "1")
    # safety net for the newest kernel on the step (persistent attention forward): checked in a throw-away process on this
    # rank's GPU before this process touches CUDA; on any failure the previous generation is pinned
    from alpa_b200.ops.selfcheck import select_attention_forward
    attn_fwd_kernel = select_attention_forward()
    torch.cuda.set_device(local_rank)

    import alpa_b200 as alpa
    from alpa_b200 import ops
    from alpa_b200.model.gpt_model import GPTModel, config_from_spec, gpt_lm_loss, gpt_train_flops, num_params
    from alpa_b200.model.model_util import TrainState, adamw, functional_call, params_of

    assert ops.native_available(), "sm_90a extension missing: run `python -c 'import __graft_entry__ as g; g.build()'`"
    # NCCL collectives that run next to compute (bucketed gradient all-reduce on its own stream) are capped to a few
    # CTAs: a full-width ring kernel next to a persistent GEMM costs the GEMM more than the reduction gains
    os.environ.setdefault("NCCL_MAX_CTAS", str(args.nccl_max_ctas))
    alpa.init(cluster="distributed" if world > 1 else "local")
    if args.nvls_allreduce < 0:
        args.nvls_allreduce = 1 if args.gpus > 1 else 0
    alpa.global_config.use_cuda_graph = bool(args.cuda_graph)
    alpa.global_config.use_nvls_grad_allreduce = bool(args.nvls_allreduce)
    alpa.global_config.use_static_grad_buckets = bool(args.grad_buckets)

    cfg = config_from_spec(args.model, dtype=torch.bfloat16)
    if args.layers is not None:
        cfg.num_hidden_layers = args.layers
    torch.manual_seed(1234)  # identical random-init weights on every rank
    model = GPTModel(cfg, device="cuda")
    params = params_of(model)

    def decay_mask(p):  # no weight decay on LayerNorm and biases (reference: weight_decay_mask)
        return {k: v.dim() > 1 for k, v in p.items()}

    state = TrainState.create(apply_fn=None, params=params, use_master_copy=True,
                              tx=adamw(1e-4, weight_decay=1e-4, mask=decay_mask, fused=True))

    def train_step(state, batch):
        def loss_fn(p):
            logits = functional_call(model, p, (batch["input_ids"], batch["position_ids"]))
            return gpt_lm_loss(logits, batch["labels"])
        loss, grads = alpa.value_and_grad(loss_fn)(state.params)
        return state.apply_gradients(grads=grads), loss

    mesh_shape = "auto" if args.mesh_shape == "auto" else tuple(int(x) for x in args.mesh_shape.lower().split("x"))
    method = {"dp": alpa.DataParallel, "zero2": alpa.Zero2Parallel, "zero3": alpa.Zero3Parallel,
              "auto": lambda: alpa.ShardParallel(logical_mesh_shape=mesh_shape)}[args.method]()
    p_step = alpa.parallelize(train_step, method=method, donate_argnums=(0,), batch_argnums=(1,))

    B = args.batch_per_gpu * args.gpus
    S = args.seq_len
    g = torch.Generator().manual_seed(7)
    host_batch = {  # pinned host memory: the e2e loop copies from here every step
        "input_ids": torch.randint(1, cfg.vocab_size, (B, S), generator=g).pin_memory(),
        "position_ids": torch.arange(S).repeat(B, 1).contiguous().pin_memory(),
        "labels": torch.randint(1, cfg.vocab_size, (B, S), generator=g).pin_memory(),
    }
    h2d_bytes = sum(t.numel() * t.element_size() for t in host_batch.values()) // args.gpus

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- warm-up (compiles: trace -> ILP -> lowering) through the e2e path
    losses = []
    for _ in range(max(3, args.warmup)):
        state, loss = p_step(state, host_batch)
        losses.append(float(loss._value))
    dev_batch = p_step.preshard_dynamic_args(state, host_batch)[1]
    executable = p_step.get_last_executable()

    if args.profile:   # per-kernel breakdown of one steady-state step (diagnostic; never a bench value)
        from torch.profiler import ProfilerActivity, profile
        barrier()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            for _ in range(2):
                state, loss = p_step(state, dev_batch)
            barrier()
        if rank == 0:
            os.makedirs(os.path.dirname(os.path.abspath(args.profile)), exist_ok=True)
            rows = [(e.key, e.count, e.device_time_total / 2e3) for e in prof.key_averages() if e.device_time_total > 0
                    and e.device_type.name == "CUDA"]
            rows.sort(key=lambda r: -r[2])
            with open(args.profile, "w") as f:
                f.write(f"# GPU kernels of one {args.model} training step (2 profiled steps averaged); ms per step\n")
                f.write(f"# total {sum(r[2] for r in rows):.2f} ms\n")
                for k, c, ms in rows:
                    f.write(f"{ms:9.3f} ms  {c // 2:5d}x  {k[:150]}\n")
        alpa.shutdown()
        return 0

    sampler = ClockSampler(local_rank)
    sampler.start()
    C = ops.native_module()

    # ---- (1) device-timed steady state: inputs resident on the device, no host round trip
    barrier()
    launches0 = C.launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.steps):
        state, loss = p_step(state, dev_batch)
    ev1.record()
    barrier()
    dev_ms = ev0.elapsed_time(ev1) / args.steps
    launches = (C.launch_count() - launches0) // args.steps

    # ---- (2) end to end: pinned-host inputs copied every step, loss read back every step
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    d2h_bytes = 0
    prev_loss = None
    e0.record()
    for _ in range(args.steps):
        state, loss = p_step(state, host_batch)
        if prev_loss is not None:            # lagged read: step i-1's loss while step i runs
            losses.append(float(prev_loss._value))
            d2h_bytes += 4
        prev_loss = loss
    losses.append(float(prev_loss._value))
    d2h_bytes += 4
    e1.record()
    barrier()
    e2e_ms = e0.elapsed_time(e1) / args.steps
    sampler.stop_flag.set()
    sampler.join(timeout=2)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, prev_loss, state)

    # max over ranks
    t = torch.tensor([dev_ms, e2e_ms], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, e2e_ms = float(t[0]), float(t[1])

    # what actually ran: the plan the ILP chose, whether the graph replay is live, how gradients were reduced
    lm_shape = tuple(int(x) for x in executable.logical_mesh.shape)
    plan = executable.plan
    sharded_inputs = sum(1 for sp in plan.input_specs.values() if sp is not None and not sp.is_replicated())
    plan_info = {"method": args.method, "logical_mesh": list(lm_shape), "ilp_objective": plan.objective,
                 "solver": plan.solver, "ilp_nodes_edge_vars": list(plan.ilp_size),
                 "sharded_inputs": sharded_inputs, "inputs": len(plan.input_specs),
                 "peak_live_bytes_per_gpu_model": getattr(plan, "peak_memory", 0.0)}
    coll = executable.count_collectives()
    dp, tp = (lm_shape + (1, 1))[:2]
    parallelism = (f"auto->dp{dp}xtp{tp}" if args.method == "auto" else f"{args.method}{args.gpus}") + \
        (f" (+{coll.get('all-to-all', 0)} a2a, {coll.get('all-gather', 0)} ag)" if coll.get("all-to-all", 0) + coll.get("all-gather", 0) else "")
    graph_live = getattr(executable, "_graph", None) not in (None, "disabled")
    kinds = sorted({getattr(b, "kind", "?") for b in executable.program.__dict__.get("_bucket_state", {}).values()})
    grad_sync = (f"{len(executable.program.grad_buckets)} static buckets: " + "/".join(kinds)) if kinds else \
        ("none (1 GPU)" if args.gpus == 1 else "per-gradient nccl")
    tokens = B * S
    flops = gpt_train_flops(B, S, cfg, backward=True, checkpoint_activations=False)
    tflops_per_gpu = flops / (dev_ms / 1e3) / args.gpus / 1e12
    peaks = {}
    try:
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "MEASURED_PEAKS.json")) as f:
            peaks = json.load(f)
    except Exception:  # noqa: BLE001
        pass
    peak = peaks.get("bf16_tflops_sustained", 989.0)   # without a measured peak: H100 SXM data-sheet dense BF16 rate
    if rank == 0:
        out = {
            "metric": "GPT-1.3B training throughput (tokens/s, whole job); PFLOPS-util in extra fields",
            "value": tokens / (dev_ms / 1e3),
            "unit": "tokens/s",
            "n_gpus": args.gpus,
            "steps": args.steps,
            "warmup": max(3, args.warmup),
            "ms_per_step": dev_ms,
            "higher_is_better": True,
            "scaling": "weak",
            "vs_baseline": tflops_per_gpu / 37.01,
            "vs_baseline_note": "TFLOPS/GPU divided by the reference's published 37.01 TFLOPS/GPU (GPT-2.6B, 8xV100, BASELINE.md)",
            "dtype": "bf16",
            "data": "synthetic random tokens, random-init weights",
            "impl": "ours",
            "tflops_per_gpu": tflops_per_gpu,
            "pflops_aggregate": tflops_per_gpu * args.gpus / 1e3,
            "pflops_util_of_measured_sustained_bf16": tflops_per_gpu / peak,
            "e2e": {"value": tokens / (e2e_ms / 1e3), "unit": "tokens/s", "ms_per_step": e2e_ms,
                    "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": d2h_bytes // args.steps,
                    "note": "per-step pinned-host -> device input copy and loss read-back (read lagged by one step)"},
            "gpu_launches": int(launches),
            "library_fallbacks": len(__import__("alpa_b200.ops.primitives", fromlist=["x"]).library_fallbacks()),
            "clocks": sampler.summary(),
            "loss_first_last": [losses[0], losses[-1]],
            "collectives_per_step": executable.count_collectives(),
            "plan": plan_info,
            "config": {"model": f"GPT-{args.model}" + ("" if args.layers is None else f"-DEBUG-{args.layers}L"),
                       "params": num_params(cfg), "global_batch": B, "seq_len": S,
                       "parallelism": parallelism, "optimizer": "AdamW fp32 master (fused)",
                       "cuda_graph": graph_live, "grad_allreduce": grad_sync,
                       "attention": "bidirectional (reference benchmark parity)",
                       "attention_fwd_kernel": attn_fwd_kernel,
                       "l2": "working set (weights 2.6 GB + activations) >> 50 MB L2; no explicit flush",
                       "flop_formula": "alpa/util.py:1658-1687, factor 72 (no remat)"},
        }
        print(json.dumps(out), flush=True)
    if world > 1:
        # all ranks are done with the timed work; skip the NCCL teardown (a communicator referenced by a captured
        # graph can block destroy_process_group) and leave with a clean exit status
        dist.barrier()
        torch.cuda.synchronize()
        sys.stdout.flush()
        os._exit(0)
    alpa.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
