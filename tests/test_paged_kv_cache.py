"""The paged KV cache without a GPU: the block allocator (`PagedKVCacheManager`), its batch layout, the paged
`ragged_attention` reference against the contiguous one, and `InputPoolConfig(kv_block_size=...)` through the pool,
`SequenceGenerator` and `LangModelWorker` against contiguous mode."""
import asyncio
import random

import pytest
import torch

from alpa_b200 import _planner, ops
from alpa_b200.model.opt_model import DecoderLM, OPTConfig
from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator


def tiny(arch="opt", **kw):
    base = dict(arch=arch, vocab_size=96, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, ffn_dim=128,
                max_position_embeddings=128, dtype=torch.float32)
    base.update(kw)
    return OPTConfig(**base)


# ------------------------------------------------------------------------------------------------------------ allocator
def test_allocator_random_invariants():
    nb, bs = 37, 4
    cm = _planner.PagedKVCacheManager(nb, bs)
    rnd = random.Random(0)
    lengths = {}
    for _ in range(2000):
        op = rnd.random()
        if op < 0.15 or not lengths:
            sid = rnd.randint(0, 10 ** 6)
            if sid not in lengths:
                cm.allocate(sid)
                lengths[sid] = 0
        elif op < 0.3:
            sid = rnd.choice(list(lengths))
            cm.free(sid)
            del lengths[sid]
        else:
            sid = rnd.choice(list(lengths))
            n = rnd.randint(0, 9)
            need = cm.blocks_needed(sid, n)
            assert need == -(-(lengths[sid] + n) // bs) - -(-lengths[sid] // bs)
            if need > cm.num_free_blocks:
                with pytest.raises(RuntimeError):
                    cm.append(sid, n)
            else:
                assert cm.append(sid, n) == lengths[sid]
                lengths[sid] += n
        owned = []
        for sid, n in lengths.items():
            table = cm.block_table(sid)
            assert len(table) == -(-n // bs) and cm.length(sid) == n
            owned += table
        assert len(owned) == len(set(owned)) and all(0 <= b < nb for b in owned)
        assert cm.num_free_blocks + len(owned) == nb and cm.num_sequences == len(lengths)


def test_allocator_errors_and_lowest_block_first():
    cm = _planner.PagedKVCacheManager(3, 2)
    cm.allocate(1)
    cm.allocate(2)
    assert cm.append(1, 3) == 0 and cm.block_table(1) == [0, 1]
    cm.append(2, 2)
    assert cm.block_table(2) == [2] and cm.num_free_blocks == 0
    cm.append(1, 1)                                   # fills the free row of block 1: no new block
    with pytest.raises(RuntimeError):
        cm.append(2, 1)
    assert cm.length(2) == 2 and cm.block_table(2) == [2]          # a failed append changes nothing
    cm.free(1)
    with pytest.raises(ValueError):
        cm.free(1)
    with pytest.raises(ValueError):
        cm.allocate(2)
    cm.allocate(3)
    cm.append(3, 1)
    assert cm.block_table(3) == [0]
    for bad in [(0, 4), (4, 0), (4, 3), (4, 2048)]:
        with pytest.raises(ValueError):
            _planner.PagedKVCacheManager(*bad)


def test_prepare_inputs_layout():
    bs = 4
    cm = _planner.PagedKVCacheManager(8, bs)
    for sid in (10, 11, 12):
        cm.allocate(sid)
    cm.append(12, 1)                                  # 12 owns block 0
    cm.append(11, 5)                                  # 11 owns blocks 1, 2 and has 5 tokens cached (a chunk ran)
    cm.append(12, 3)                                  # 12 fills block 0 without a new block
    out = cm.prepare_inputs([10, 11], [3, 4], [12], 12, 99, [False, True], 6)
    assert out["num_tokens"] == 8
    # sequence 10: a first chunk of 3 tokens (block 3); 11 continues at position 5 (block 2 rows 1-3, then block 4);
    # 12 decodes at position 4 (block 5)
    assert out["block_table"] == [[3, 0, 0, 0, 0, 0], [1, 2, 4, 0, 0, 0], [0, 5, 0, 0, 0, 0]]
    assert out["slot"] == [12, 13, 14, 9, 10, 11, 16, 20, 99, 99, 99, 99]
    assert out["seq_start"] == [0, 0, 0, 1, 1, 1, 1, 2, 0, 0, 0, 0]
    assert out["position"] == [0, 1, 2, 5, 6, 7, 8, 4, 0, 0, 0, 0]
    assert out["ctx_len"] == [1, 2, 3, 6, 7, 8, 9, 5, 0, 0, 0, 0]
    assert out["logit_index"] == [6, 7]                # 10's chunk does not end its prefill
    for t in range(8):
        row = out["block_table"][out["seq_start"][t]]
        pos = out["position"][t]
        assert out["slot"][t] == row[pos // bs] * bs + pos % bs
    assert cm.length(10) == 3 and cm.length(11) == 9 and cm.length(12) == 5
    with pytest.raises(RuntimeError):                 # 2 blocks left, 3 needed: nothing is taken
        cm.prepare_inputs([10], [12], [], 16, 99)
    assert cm.num_free_blocks == 2 and cm.length(10) == 3


# ------------------------------------------------------------------------------------------------------- reference op
def _paged_case(seed, h=4, hkv=2, D=16, bs=4, lens=(9, 1, 14), fp8=False):
    """Sequences of `lens` keys in shuffled blocks interleaved between sequences, and the same keys gathered into
    consecutive rows of a contiguous cache.  Each sequence's tokens are its last 2 positions (one when it has one)."""
    g = torch.Generator().manual_seed(seed)
    nblk = sum(-(-n // bs) for n in lens) + 3
    slots = nblk * bs + 1
    perm = torch.randperm(nblk, generator=g).tolist()
    data_k = torch.randn(slots, hkv, D, generator=g).bfloat16().float()
    data_v = torch.randn(slots, hkv, D, generator=g).bfloat16().float()
    width = max(-(-n // bs) for n in lens) + 1
    table, gather, starts, ss, sp, cl = [], [], [], [], [], []
    for i, n in enumerate(lens):
        blocks = [perm.pop() for _ in range(-(-n // bs))]
        table.append(blocks + [0] * (width - len(blocks)))
        starts.append(len(gather))
        gather += [blocks[j // bs] * bs + j % bs for j in range(n)]
        for j in range(max(0, n - 2), n):
            ss.append(i)
            sp.append(starts[i])
            cl.append(j + 1)
    ss.append(0), sp.append(0), cl.append(0)          # a padding token
    T = len(cl)
    q = torch.randn(T, h, D, generator=g).bfloat16().float()
    idx = torch.tensor(gather + [slots - 1])          # the contiguous copy keeps a scratch row last
    kc, vc = data_k[idx], data_v[idx]
    if fp8:
        pk, pv = ops.Fp8KV.zeros((slots, hkv, D), "cpu"), ops.Fp8KV.zeros((slots, hkv, D), "cpu")
        P = ops.primitives
        P._kv_store_ref(data_k[None], data_v[None], pk, pv, 0, torch.arange(slots))
        rows = lambda c: ops.Fp8KV(c.data.view(torch.uint8)[idx].view(torch.float8_e4m3fn), c.scale[:, idx])  # noqa: E731
        ck, cv = rows(pk), rows(pv)
        data_k, data_v, kc, vc = pk, pv, ck, cv
    bt = torch.tensor(table, dtype=torch.int32)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32)  # noqa: E731
    return q, data_k, data_v, kc, vc, bt, i32(ss), i32(sp), i32(cl), width * bs


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("alibi", [False, True])
def test_paged_reference_equals_contiguous_on_gathered_cache(fp8, alibi):
    q, pk, pv, ck, cv, bt, ss, sp, cl, mc = _paged_case(1, fp8=fp8)
    ab = torch.tensor([0.5, 0.25, 0.125, 0.0625]) if alibi else None
    got = ops.primitives.ragged_attention(q, pk, pv, ss, cl, 0.25, mc, ab, bt, 4)
    want = ops.primitives.ragged_attention(q, ck, cv, sp, cl, 0.25, mc, ab)
    assert torch.equal(got, want)
    assert bool((got[cl == 0] == 0).all()) and bool(got[cl > 0].abs().sum() > 0)


def test_paged_reference_rejects_out_of_range_entries():
    q, pk, pv, ck, cv, bt, ss, sp, cl, mc = _paged_case(2)
    nblk = (pk.shape[0] - 1) // 4
    for bad in (nblk, -1):
        t = bt.clone()
        t[0, 0] = bad
        with pytest.raises(ValueError):
            ops.primitives.ragged_attention(q, pk, pv, ss, cl, 0.25, mc, None, t, 4)
    t = bt.clone()
    t[0, -1] = nblk + 5                               # an entry past the sequence's keys is never read
    ops.primitives.ragged_attention(q, pk, pv, ss, cl, 0.25, mc, None, t, 4)
    with pytest.raises(ValueError):
        ops.primitives.ragged_attention(q, pk, pv, ss, cl, 0.25, mc, None, bt, 3)
    with pytest.raises(ValueError):
        ops.primitives.ragged_attention(q, pk, pv, ss, cl, 0.25, mc, None, bt)


# ---------------------------------------------------------------------------------------------------------------- pool
def _drain(pool, rnd_tokens=7):
    """Run a pool to completion with a fake model that emits token `rnd_tokens` (never end-of-sequence); returns the
    most sequences that produced a token in one iteration."""
    most = 0
    while not pool.is_finished():
        b = pool.next()
        most = max(most, len(b["logit_index"]))
        pool.update([rnd_tokens] * len(b["logit_index"]))
    return most


def test_paged_pool_runs_more_sequences_than_contiguous():
    # 8 prompts of 4 tokens that each stop after 4 new tokens, declared cap 32: contiguous reserves 32 slots each, so
    # a 64-slot cache runs 2 at a time; paged needs at most 8 tokens = 2 blocks of 4 each, so all 8 run together
    prompts = [[5, 6, 7, 8]] * 8
    counts = {}
    for bs in (None, 4):
        cfg = InputPoolConfig(batch_size=64, cache_size=64, max_cache_per_seq=32, pad_multiple=8, kv_block_size=bs)
        pool = IterationLevelInputPool(cfg, max_new_tokens=4)
        pool.enter_prompts(prompts, max_lengths=[32] * 8)
        counts[bs] = _drain(pool)
        assert len(pool.get_results()) == 8 and all(len(r) == 8 for r in pool.get_results())
    assert counts == {None: 2, 4: 8}
    assert pool.num_preemptions == 0 and pool.peak_blocks_used == 16


def test_paged_pool_preempts_when_blocks_run_out_and_finishes():
    cfg = InputPoolConfig(batch_size=32, cache_size=32, max_cache_per_seq=32, pad_multiple=8, kv_block_size=4)
    pool = IterationLevelInputPool(cfg, max_new_tokens=12)
    pool.enter_prompts([[3 + i] * 5 for i in range(4)])
    _drain(pool)
    assert pool.num_preemptions > 0 and pool.peak_blocks_used <= 8
    res = pool.get_results()
    assert len(res) == 4 and all(len(r) == 17 for r in res)
    assert pool.cache_manager.num_free_blocks == 8


def test_paged_pool_prefills_long_prompt_in_chunks():
    cfg = InputPoolConfig(batch_size=8, cache_size=64, max_cache_per_seq=40, pad_multiple=8, kv_block_size=8)
    pool = IterationLevelInputPool(cfg, max_new_tokens=2)
    pool.enter_prompts([list(range(3, 23))])            # 20 tokens, 8 per iteration
    b = pool.next()
    assert b["ctx_len"] == list(range(1, 9)) and b["logit_index"] == []
    pool.update([])
    b = pool.next()
    assert b["position"] == list(range(8, 16)) and b["logit_index"] == []
    pool.update([])
    b = pool.next()
    assert b["position"][:4] == list(range(16, 20)) and b["logit_index"] == [3]
    pool.update([9])
    _drain(pool)
    assert pool.get_results() == [list(range(3, 23)) + [9, 7]]


def test_paged_pool_config_errors():
    with pytest.raises(ValueError):
        IterationLevelInputPool(InputPoolConfig(cache_size=100, kv_block_size=16))
    with pytest.raises(ValueError):
        IterationLevelInputPool(InputPoolConfig(cache_size=96, kv_block_size=12))
    pool = IterationLevelInputPool(InputPoolConfig(batch_size=8, cache_size=32, max_cache_per_seq=64, kv_block_size=8))
    with pytest.raises(ValueError):
        pool.enter_prompts([[4] * 32])                  # no room to generate in the cache
    pool.enter_prompts([[4] * 20])                      # longer than the token budget: chunked, not rejected
    assert pool.todo[0].max_length == 32
    contiguous = IterationLevelInputPool(InputPoolConfig(batch_size=8, cache_size=32, max_cache_per_seq=16))
    with pytest.raises(ValueError):
        contiguous.enter_prompts([[4] * 9])
    assert pool.accepts_prompt(20) and not contiguous.accepts_prompt(9) and contiguous.accepts_prompt(8)


# ---------------------------------------------------------------------------------------------------------- end to end
def _prompts(seed, n=6, lo=2, hi=9, V=96):
    rnd = random.Random(seed)
    return [[rnd.randint(3, V - 1) for _ in range(rnd.randint(lo, hi))] for _ in range(n)]


def _model(arch, cache):
    kw = {"num_key_value_heads": 2} if arch == "llama" else {}
    return DecoderLM(tiny(arch, kv_cache_dtype=cache, **kw), device="cpu", seed=3)


@pytest.mark.parametrize("arch", ["opt", "llama"])
@pytest.mark.parametrize("cache", ["bf16", "fp8"])
def test_paged_generation_equals_contiguous(arch, cache):
    m = _model(arch, cache)
    prompts = _prompts(7)
    want = SequenceGenerator(m, InputPoolConfig(batch_size=32, cache_size=96, max_cache_per_seq=24)).generate(
        prompts, max_new_tokens=10)
    # roomy: no preemption; tight: preemption and recompute; small budget: chunked prefill
    for cfg, preempts in [(InputPoolConfig(batch_size=32, cache_size=96, max_cache_per_seq=24, kv_block_size=4), 0),
                          (InputPoolConfig(batch_size=32, cache_size=40, max_cache_per_seq=24, kv_block_size=4), 1),
                          (InputPoolConfig(batch_size=8, cache_size=64, max_cache_per_seq=24, kv_block_size=2), None)]:
        gen = SequenceGenerator(m, cfg)
        pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                       max_new_tokens=10)
        pool.enter_prompts(prompts)
        while not pool.is_finished():
            gen.step(pool)
        assert pool.get_results() == want, cfg
        if preempts is not None:
            assert (pool.num_preemptions > 0) == bool(preempts), cfg


def _logits_by_step(m, cfg, prompts, new_tokens=5):
    """{(sequence id, generated count): logits} of a run whose sampler forces a fixed token per (sequence, step), so
    every mode sees the same sequences whatever its logits, plus the pool."""
    gen = SequenceGenerator(m, cfg)
    pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                   max_new_tokens=new_tokens)
    pool.enter_prompts(prompts)
    seen = {}

    def forced(logits):
        rows = pool._current
        for r, p in enumerate(rows):
            seen[(p.sentence_id, p.generation_length)] = logits[r].clone()
        return torch.tensor([3 + (7 * p.sentence_id + 5 * p.generation_length) % 90 for p in rows])
    while not pool.is_finished():
        gen.step(pool, forced)
    return seen, pool


@pytest.mark.parametrize("arch", ["opt", "llama"])
@pytest.mark.parametrize("cache", ["bf16", "fp8"])
def test_chunked_and_preempted_logits_equal_contiguous(arch, cache):
    """Every logit row of paged runs with chunk-only iterations (prompts longer than the token budget, no decoder
    running) and with preemption and recompute against contiguous mode.  A chunk whose K/V were not written would
    shift these logits by about 0.1; float32 row-order rounding stays below 1e-4."""
    m = _model(arch, cache)
    prompts = _prompts(11, n=3, lo=23, hi=27)
    base = InputPoolConfig(batch_size=96, cache_size=128, max_cache_per_seq=40)
    want, _ = _logits_by_step(m, base, prompts)
    for cfg, what in [(InputPoolConfig(batch_size=16, cache_size=128, max_cache_per_seq=40, kv_block_size=8), "chunk"),
                      (InputPoolConfig(batch_size=96, cache_size=64, max_cache_per_seq=40, kv_block_size=4), "preempt")]:
        got, pool = _logits_by_step(m, cfg, prompts)
        assert got.keys() == want.keys(), what
        if what == "preempt":
            assert pool.num_preemptions > 0
        scale = max(float(v.abs().max()) for v in want.values())
        err = max(float((got[k] - want[k]).abs().max()) for k in want)
        assert err <= 1e-4 * max(1.0, scale), (what, err, scale)


def test_chunk_only_iteration_writes_the_cache():
    """The first iteration of a prompt longer than the token budget has no logit row; the model must still run."""
    m = _model("opt", "bf16")
    cfg = InputPoolConfig(batch_size=16, cache_size=128, max_cache_per_seq=40, kv_block_size=8)
    gen = SequenceGenerator(m, cfg)
    pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, max_new_tokens=2)
    pool.enter_prompts([list(range(3, 26))])
    k0 = gen.cache[0][0].clone()
    assert gen.step(pool) == 0 and gen.iterations == 1
    written = (gen.cache[0][0] != k0).flatten(1).any(1)
    assert written[:16].all() and not written[16:].any()


def test_model_worker_paged_equals_contiguous():
    from alpa_b200.serve.model_worker import LangModelWorker
    m = _model("opt", "bf16")
    prompts = _prompts(9, n=8)
    limits = [random.Random(i).randint(1, 8) for i in range(8)]

    async def serve(cfg):
        w = LangModelWorker(m, cfg)
        res = await asyncio.wait_for(asyncio.gather(*[w.completions(p, n) for p, n in zip(prompts, limits)]), 120)
        await w.shutdown()
        return [r["ids"] for r in res], w

    want, _ = asyncio.run(serve(InputPoolConfig(batch_size=16, cache_size=48, max_cache_per_seq=16)))
    got, w = asyncio.run(serve(InputPoolConfig(batch_size=16, cache_size=48, max_cache_per_seq=16, kv_block_size=4)))
    assert got == want
    assert w.pool.cache_manager.num_free_blocks == 12
