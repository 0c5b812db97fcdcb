"""Multi-LoRA serving on the CPU (PyTorch references of ops.lora_shrink / ops.lora_expand_): adapters loaded next to one
base model, selected per request in continuous batching, against models built from merged weights."""
import asyncio
import json
import os
import sys

import numpy as np
import pytest
import torch

from alpa_b200.model.gpt_model import llama_params_from_hf
from alpa_b200.model.opt_model import DecoderLM, OPTConfig, gpt_config_from_serving
from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator
from alpa_b200.serve.generator import load_lora_np
from alpa_b200.serve.model_worker import LangModelWorker

V, H, NH, I, L = 96, 64, 4, 128, 2
LLAMA_MODS = {"q_proj": "self_attn", "k_proj": "self_attn", "v_proj": "self_attn", "o_proj": "self_attn",
              "gate_proj": "mlp", "up_proj": "mlp", "down_proj": "mlp"}
OPT_MODS = {"q_proj": "self_attn", "k_proj": "self_attn", "v_proj": "self_attn", "out_proj": "self_attn", "fc2": ""}


def tiny(arch, **kw):
    base = dict(arch=arch, vocab_size=V, hidden_size=H, num_hidden_layers=L, num_attention_heads=NH, ffn_dim=I,
                max_position_embeddings=256, dtype=torch.float32, max_loras=4, max_lora_rank=16)
    if arch == "llama":
        base.update(num_key_value_heads=2, activation="silu", pad_token_id=0)
    base.update(kw)
    return OPTConfig(**base)


def _shapes(cfg, mod):
    """(in, out) of a module in Hugging Face's layout."""
    D, kv, H, I = cfg.head_dim, cfg.kv_heads, cfg.hidden_size, cfg.ffn_dim
    return {"q_proj": (H, cfg.num_attention_heads * D), "k_proj": (H, kv * D), "v_proj": (H, kv * D), "o_proj": (H, H),
            "out_proj": (H, H), "gate_proj": (H, I), "up_proj": (H, I), "down_proj": (I, H), "fc2": (I, H)}[mod]


def _base_hf(cfg, seed):
    """Random base weights under Hugging Face names (Llama) or DecoderLM's OPT parameter names."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g) * 0.05  # noqa: E731
    V, H, NH, I, L = cfg.vocab_size, cfg.hidden_size, cfg.num_attention_heads, cfg.ffn_dim, cfg.num_hidden_layers
    if cfg.arch == "llama":
        sd = {"embed_tokens.weight": rnd(V, H), "norm.weight": 1 + rnd(H), "lm_head.weight": rnd(V, H)}
        for i in range(L):
            p = f"layers.{i}."
            sd[p + "input_layernorm.weight"] = 1 + rnd(H)
            sd[p + "post_attention_layernorm.weight"] = 1 + rnd(H)
            for mod, blk in LLAMA_MODS.items():
                k_in, n_out = _shapes(cfg, mod)
                sd[f"{p}{blk}.{mod}.weight"] = rnd(n_out, k_in)
        return sd
    D = cfg.head_dim
    p = {"embed_tokens": rnd(V, H), "embed_positions": rnd(256 + 2, H)}
    for i in range(L):
        p[f"layers.{i}.qkv.w"] = rnd(3, NH, D, H)
        p[f"layers.{i}.out.w"] = rnd(H, H)
        p[f"layers.{i}.fc1.w"] = rnd(I, H)
        p[f"layers.{i}.fc2.w"] = rnd(H, I)
    return p


def _params(cfg, base, merged=None):
    """DecoderLM params of `base` with each (layer, module) weight plus its delta in `merged` (s * B A)."""
    merged = merged or {}
    if cfg.arch == "llama":
        sd = dict(base)
        for (i, mod), d in merged.items():
            k = f"layers.{i}.{LLAMA_MODS[mod]}.{mod}.weight"
            sd[k] = sd[k] + d
        return llama_params_from_hf(sd, gpt_config_from_serving(cfg))
    p = {k: v.clone() for k, v in base.items()}
    D, NH, H = cfg.head_dim, cfg.num_attention_heads, cfg.hidden_size
    for (i, mod), d in merged.items():
        if mod in ("q_proj", "k_proj", "v_proj"):
            p[f"layers.{i}.qkv.w"][("q_proj", "k_proj", "v_proj").index(mod)] += d.view(NH, D, H)
        else:
            p[f"layers.{i}.{'out' if mod == 'out_proj' else 'fc2'}.w"] += d
    return p


def _adapter(cfg, path, r, alpha, seed, mods=None):
    """Write a PEFT adapter directory (.npy per tensor); returns {(layer, module): s * B A}."""
    mods = mods or list(LLAMA_MODS if cfg.arch == "llama" else OPT_MODS)
    os.makedirs(path, exist_ok=True)
    g = torch.Generator().manual_seed(seed)
    deltas = {}
    prefix = "base_model.model.model." + ("" if cfg.arch == "llama" else "decoder.")
    blocks = LLAMA_MODS if cfg.arch == "llama" else OPT_MODS
    for i in range(cfg.num_hidden_layers):
        for mod in mods:
            k_in, n_out = _shapes(cfg, mod)
            A, B = torch.randn(r, k_in, generator=g) * 0.2, torch.randn(n_out, r, generator=g) * 0.2
            name = f"{prefix}layers.{i}.{blocks[mod] + '.' if blocks[mod] else ''}{mod}"
            np.save(os.path.join(path, name + ".lora_A.weight.npy"), A.numpy())
            np.save(os.path.join(path, name + ".lora_B.weight.npy"), B.numpy())
            deltas[(i, mod)] = (alpha / r) * (B @ A)
    with open(os.path.join(path, "adapter_config.json"), "w") as f:
        json.dump({"r": r, "lora_alpha": alpha, "target_modules": mods}, f)
    return deltas


def _run(m, prompts, loras, pool_cfg, steps=4):
    """{(prompt index, generated count): logits} with a forced token per (sequence, step), so runs whose logits differ
    in the last bits still feed the same tokens."""
    gen = SequenceGenerator(m, pool_cfg)
    pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                   max_new_tokens=steps, model=m)
    sids = pool.enter_prompts(prompts, loras=[None if n is None else m.lora_id(n) for n in loras])
    index = {sid: k for k, sid in enumerate(sids)}
    seen = {}

    def sampler(logits):
        out = []
        for row, p in enumerate(pool._current):
            seen[(index[p.sentence_id], p.generation_length)] = logits[row].clone()
            out.append(3 + (p.sentence_id * 7 + p.generation_length * 5) % (m.cfg.vocab_size - 3))
        return torch.tensor(out)
    while not pool.is_finished():
        gen.step(pool, sampler)
    return seen, pool


def _prompts(n, seed, lo=5, hi=30, V=V):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(3, V, (int(torch.randint(lo, hi, (1,), generator=g)),), generator=g).tolist()
            for _ in range(n)]


POOLS = {"contiguous": dict(batch_size=128, cache_size=1024, max_cache_per_seq=64),
         "paged": dict(batch_size=48, cache_size=512, max_cache_per_seq=64, kv_block_size=16),
         "prefix": dict(batch_size=48, cache_size=512, max_cache_per_seq=64, kv_block_size=16, prefix_caching=True)}


@pytest.mark.parametrize("pool", list(POOLS))
@pytest.mark.parametrize("arch", ["llama", "opt"])
def test_merged_weight_oracle_and_base_rows_untouched(tmp_path, arch, pool):
    cfg = tiny(arch)
    base = _base_hf(cfg, 1)
    m = DecoderLM(cfg, device="cpu", params=_params(cfg, base))
    mods = list(LLAMA_MODS if arch == "llama" else OPT_MODS)
    # mixed ranks, one adapter with only some targets
    specs = {"a": (4, 8.0, None), "b": (16, 16.0, None), "c": (8, 32.0, mods[::2])}
    deltas = {}
    for k, (name, (r, alpha, sub)) in enumerate(specs.items()):
        deltas[name] = _adapter(cfg, str(tmp_path / name), r, alpha, 10 + k, sub)
        m.load_lora(name, *load_lora_np(cfg, str(tmp_path / name)))
    prompts = _prompts(8, 2)
    loras = [None, "a", "b", None, "c", "a", "b", "c"]
    pc = InputPoolConfig(**POOLS[pool])
    got, _ = _run(m, prompts, loras, pc)
    base_only, _ = _run(m, prompts, [None] * 8, InputPoolConfig(**POOLS[pool]))
    for name in specs:
        merged = DecoderLM(cfg, device="cpu", params=_params(cfg, base, deltas[name]))
        want, _ = _run(merged, prompts, [None] * 8, InputPoolConfig(**POOLS[pool]))
        for key, lg in got.items():
            if loras[key[0]] == name:
                torch.testing.assert_close(lg, want[key], atol=2e-4, rtol=1e-4)
    for key, lg in got.items():
        if loras[key[0]] is None:
            assert torch.equal(lg, base_only[key]), key
        else:
            assert not torch.allclose(lg, base_only[key], atol=1e-3), key


def test_preempted_sequence_keeps_its_adapter(tmp_path):
    cfg = tiny("llama")
    base = _base_hf(cfg, 1)
    m = DecoderLM(cfg, device="cpu", params=_params(cfg, base))
    deltas = _adapter(cfg, str(tmp_path / "a"), 8, 16.0, 3)
    m.load_lora("a", *load_lora_np(cfg, str(tmp_path / "a")))
    merged = DecoderLM(cfg, device="cpu", params=_params(cfg, base, deltas))
    prompts = _prompts(6, 4, 20, 30)
    tight = dict(batch_size=64, cache_size=160, max_cache_per_seq=64, kv_block_size=16)
    got, pool = _run(m, prompts, ["a"] * 6, InputPoolConfig(**tight), steps=12)
    assert pool.num_preemptions > 0
    want, _ = _run(merged, prompts, [None] * 6, InputPoolConfig(**tight), steps=12)
    assert got.keys() == want.keys()
    for key in got:
        torch.testing.assert_close(got[key], want[key], atol=2e-4, rtol=1e-4)


def _finish(pool, m, prompt, lora):
    """Serve one prompt to its end; returns the prefix-cache hit tokens of its admission."""
    gen = SequenceGenerator(m, pool.config)
    before = pool.prefix_hit_tokens
    pool.enter_prompts([prompt], loras=[None if lora is None else m.lora_id(lora)])
    while not pool.is_finished():
        gen.step(pool)
    return pool.prefix_hit_tokens - before


def test_prefix_cache_blocks_never_cross_adapters(tmp_path):
    cfg = tiny("llama")
    m = DecoderLM(cfg, device="cpu", seed=3)
    for name, seed in (("a", 1), ("b", 2)):
        _adapter(cfg, str(tmp_path / name), 8, 8.0, seed)
        m.load_lora(name, *load_lora_np(cfg, str(tmp_path / name)))
    pc = InputPoolConfig(**POOLS["prefix"])
    pool = IterationLevelInputPool(pc, pad_token_id=0, eos_token_id=2, max_new_tokens=2, model=m)
    prompt = _prompts(1, 5, 40, 41)[0]
    assert _finish(pool, m, prompt, "a") == 0
    assert _finish(pool, m, prompt, "b") == 0            # same tokens, another adapter: no block shared
    assert _finish(pool, m, prompt, None) == 0           # nor with the base model
    assert _finish(pool, m, prompt, "a") == 32           # same adapter: the full blocks before the last token
    assert _finish(pool, m, prompt, None) == 32
    m.unload_lora("a")
    m.load_lora("a", *load_lora_np(cfg, str(tmp_path / "a")))
    assert _finish(pool, m, prompt, "a") == 0            # a reloaded adapter has a new load id


def test_namespace_zero_keeps_the_base_keys():
    from alpa_b200 import _planner
    rng = np.random.default_rng(0)
    toks = [rng.integers(3, 90, 70).tolist() for _ in range(3)]
    hits = []
    for explicit in (False, True):
        cm = _planner.PagedKVCacheManager(32, 16, True)
        kw = {"namespace": 0} if explicit else {}
        got = []
        for sid, t in enumerate(toks + toks, 1):
            got.append(cm.match_prefix(sid, t, **kw))
            cm.prepare_inputs([sid], [len(t) - got[-1]], [], 128, 512, [True], 8, t[got[-1]:])
            cm.free(sid)
        hits.append((got, cm.num_cached_blocks))
    assert hits[0] == hits[1] and hits[0][0][3:] == [64, 64, 64]
    cm = _planner.PagedKVCacheManager(32, 16, True)
    cm.allocate(1, namespace=7)
    cm.prepare_inputs([1], [40], [], 128, 512, [True], 8, toks[0][:40])
    cm.free(1)
    assert cm.match_prefix(2, toks[0][:40], namespace=0) == 0 and cm.match_prefix(3, toks[0][:40], namespace=7) == 32
    with pytest.raises(ValueError):
        cm.allocate(4, namespace=-1)


def test_errors(tmp_path):
    cfg = tiny("opt", max_loras=2, max_lora_rank=8)
    m = DecoderLM(cfg, device="cpu", seed=1)
    _adapter(cfg, str(tmp_path / "a"), 8, 8.0, 1)
    t = load_lora_np(cfg, str(tmp_path / "a"))
    assert m.load_lora("a", *t) == 0 and m.load_lora("b", *t) == 1
    with pytest.raises(ValueError, match="slots are taken"):
        m.load_lora("c", *t)
    with pytest.raises(ValueError, match="already loaded"):
        m.load_lora("a", *t)
    m.unload_lora("b")
    with pytest.raises(ValueError, match="rank"):
        m.load_lora("big", t[0], 8.0, 16)
    fc1 = {"base_model.model.model.decoder.layers.0.fc1.lora_A.weight": torch.zeros(8, H),
           "base_model.model.model.decoder.layers.0.fc1.lora_B.weight": torch.zeros(I, 8)}
    with pytest.raises(ValueError, match="not a supported LoRA target"):
        m.load_lora("fc1", fc1, 8.0, 8)
    with open(tmp_path / "a" / "adapter_config.json", "w") as f:
        json.dump({"r": 8, "lora_alpha": 8, "target_modules": ["q_proj", "fc1"]}, f)
    with pytest.raises(ValueError, match="fc1"):
        load_lora_np(cfg, str(tmp_path / "a"))
    with pytest.raises(ValueError, match="Llama and OPT"):
        DecoderLM(tiny("bloom"), device="cpu").load_lora("x", {}, 1.0, 1)
    with pytest.raises(ValueError, match="Llama and OPT"):
        DecoderLM(tiny("codegen", rotary_dim=8), device="cpu").load_lora("x", {}, 1.0, 1)
    with pytest.raises(ValueError, match="unknown LoRA"):
        m.lora_id("b")
    # in use while a prompt of a pool is queued or running
    pool = IterationLevelInputPool(InputPoolConfig(**POOLS["paged"]), model=m, max_new_tokens=3)
    pool.enter_prompts([[5, 6, 7]], loras=[m.lora_id("a")])
    with pytest.raises(RuntimeError, match="in use"):
        m.unload_lora("a")
    gen = SequenceGenerator(m, pool.config)
    gen.step(pool)
    with pytest.raises(RuntimeError, match="in use"):
        m.unload_lora("a")
    while not pool.is_finished():
        gen.step(pool)
    m.unload_lora("a")
    with pytest.raises(ValueError):
        pool.enter_prompts([[5, 6, 7]], loras=[12345])


def test_worker_lora_requests(tmp_path):
    cfg = tiny("llama")
    base = _base_hf(cfg, 1)
    m = DecoderLM(cfg, device="cpu", params=_params(cfg, base))
    deltas = _adapter(cfg, str(tmp_path / "a"), 8, 16.0, 3)
    m.load_lora("a", *load_lora_np(cfg, str(tmp_path / "a")))
    merged = DecoderLM(cfg, device="cpu", params=_params(cfg, base, deltas))

    async def go(model, req):
        w = LangModelWorker(model, InputPoolConfig(**POOLS["paged"]))
        try:
            return await w.handle_request(req)
        finally:
            await w.shutdown()
    prompt = [5, 9, 11, 20, 31, 7]
    got = asyncio.run(go(m, {"prompt_ids": prompt, "max_tokens": 6, "lora": "a"}))
    want = asyncio.run(go(merged, {"prompt_ids": prompt, "max_tokens": 6}))
    assert got["ids"] == want["ids"]
    lp = asyncio.run(go(m, {"prompt_ids": prompt, "logprobs": True, "lora": "a"}))
    lp_want = asyncio.run(go(merged, {"prompt_ids": prompt, "logprobs": True}))
    np.testing.assert_allclose(lp["token_logprobs"][1:], lp_want["token_logprobs"][1:], atol=1e-4)
    with pytest.raises(ValueError, match="unknown LoRA"):
        asyncio.run(go(m, {"prompt_ids": prompt, "max_tokens": 2, "lora": "nope"}))


def _tp_worker(rank, world, port, tmp):
    """One rank of the tensor-parallel check: Llama (Hkv = 2) and OPT with adapters served with tp = world give the
    logits of tp = 1."""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        for arch in ("llama", "opt"):
            cfg = tiny(arch)
            path = os.path.join(tmp, f"{arch}{rank}")
            _adapter(cfg, path, 8, 16.0, 4)
            prompts = _prompts(4, 6)
            outs = []
            for group in (None, dist.group.WORLD):
                m = DecoderLM(cfg, device="cpu", group=group, seed=5)
                m.load_lora("a", *load_lora_np(cfg, path))
                outs.append(_run(m, prompts, ["a", None, "a", "a"], InputPoolConfig(**POOLS["paged"]))[0])
            assert outs[0].keys() == outs[1].keys()
            for k in outs[0]:
                torch.testing.assert_close(outs[0][k], outs[1][k], atol=2e-4, rtol=1e-4)
        print(f"rank {rank}: lora tp ok", flush=True)
    finally:
        dist.destroy_process_group()


def test_tensor_parallel_world2(tmp_path):
    import socket
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    code = ("import sys; sys.path[:0] = [{!r}, {!r}]; import test_lora_serving as t; t._tp_worker({{}}, 2, {}, {!r})"
            .format(os.path.dirname(here), here, port, str(tmp_path)))
    procs = [subprocess.Popen([sys.executable, "-c", code.format(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    try:
        outs = [p.communicate(timeout=300)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r}: lora tp ok" in out, out
