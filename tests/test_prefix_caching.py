"""Prefix caching for the paged KV cache without a GPU: the block manager's index, reference counts and eviction, the
paged prefill reference op, and `InputPoolConfig(prefix_caching=True)` through the pool, `SequenceGenerator` and
`LangModelWorker` against caching off."""
import asyncio
import random

import pytest
import torch

from alpa_b200 import _planner, ops
from alpa_b200.model.opt_model import DecoderLM, OPTConfig
from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator

BS = 16


def _fill(cm, sid, tokens, batch=4096):
    """Allocate `sid` from the cache's matching prefix and lay out the rest of `tokens` in one prefill; returns the
    hit and the prepare_inputs result."""
    hit = cm.match_prefix(sid, tokens)
    out = cm.prepare_inputs([sid], [len(tokens) - hit], [], batch, 0, [], 0, tokens[hit:])
    return hit, out


# ------------------------------------------------------------------------------------------------------------- manager
def test_match_is_exact_even_when_every_hash_collides():
    cm = _planner.PagedKVCacheManager(16, BS, True, 1)          # a 1-bit hash: unequal blocks collide
    a = list(range(100, 100 + 2 * BS + 5))
    _fill(cm, 1, a)
    assert cm.num_cached_blocks == 2                           # 37 tokens laid out: the first two blocks are full
    b = a[:BS] + [7] + a[BS + 1:]                              # one token differs in block 1
    assert cm.match_prefix(2, b) == BS
    c = [a[0] + 1] + a[1:]                                     # differs in block 0: nothing chains
    assert cm.match_prefix(3, c) == 0
    # the same token ids after a different prefix are a different key
    d = [9] * BS + a[BS:2 * BS] + [1]
    assert cm.match_prefix(4, d) == 0


@pytest.mark.parametrize("n,cap", [(1, 0), (BS - 1, 0), (BS, 0), (BS + 1, BS), (2 * BS, BS), (2 * BS + 1, 2 * BS)])
def test_hit_leaves_at_least_one_token(n, cap):
    cm = _planner.PagedKVCacheManager(16, BS, True)
    toks = list(range(3, 3 + 3 * BS))
    _fill(cm, 1, toks)
    assert cm.match_prefix(2, toks[:n]) == cap
    assert cm.length(2) == cap and len(cm.block_table(2)) == cap // BS


def test_refcounts_through_sharing_release_and_preemption():
    cm = _planner.PagedKVCacheManager(8, BS, True)
    toks = list(range(2 * BS + 3))
    _fill(cm, 1, toks)
    shared = cm.block_table(1)[:2]
    assert [cm.ref_count(b) for b in shared] == [1, 1] and all(cm.is_cached(b) for b in shared)
    assert cm.match_prefix(2, toks) == 2 * BS and cm.block_table(2) == shared
    assert cm.match_prefix(3, toks[:BS + 1]) == BS
    assert [cm.ref_count(b) for b in shared] == [3, 2]
    free = cm.num_free_blocks
    cm.free(1)                                                # 1's partial block 2 goes back to the free set
    assert [cm.ref_count(b) for b in shared] == [2, 1] and cm.num_free_blocks == free + 1
    cm.free(2)
    cm.free(3)                                                # a preemption: all references dropped, content kept
    assert [cm.ref_count(b) for b in shared] == [0, 0]
    assert cm.num_evictable_blocks == 2 and cm.num_free_blocks == 8 and cm.num_cached_blocks == 2
    assert cm.match_prefix(4, toks) == 2 * BS                 # re-admission before eviction: both blocks hit
    assert cm.num_evictable_blocks == 0 and cm.num_free_blocks == 6
    with pytest.raises(RuntimeError):
        cm.reset_prefix_cache()                               # a sequence is live
    cm.free(4)
    cm.reset_prefix_cache()
    assert cm.num_cached_blocks == 0 and cm.num_free_blocks == 8 and cm.match_prefix(5, toks) == 0


def test_eviction_takes_uncached_blocks_first_then_lru():
    cm = _planner.PagedKVCacheManager(4, BS, True)
    x, y = [5] * BS + [1], [6] * BS + [1]
    _fill(cm, 1, x)                                           # blocks 0 (cached), 1
    _fill(cm, 2, y)                                           # blocks 2 (cached), 3
    bx, by = cm.block_table(1)[0], cm.block_table(2)[0]
    cm.free(2)                                                # y released first: the least recently released
    cm.free(1)
    assert cm.num_free_blocks == 4 and cm.num_evictable_blocks == 2
    cm.allocate(3)
    cm.append(3, 2 * BS)                                      # takes the two uncached blocks first
    assert sorted(cm.block_table(3)) == sorted({0, 1, 2, 3} - {bx, by}) and cm.num_cached_blocks == 2
    cm.append(3, 1)                                           # now evicts y's block
    assert cm.block_table(3)[-1] == by and cm.num_cached_blocks == 1
    assert cm.match_prefix(4, y) == 0 and cm.match_prefix(5, x) == BS


def test_evicted_parent_makes_children_unmatchable():
    cm = _planner.PagedKVCacheManager(6, BS, True)
    a0, a1, b1 = list(range(10, 10 + BS)), list(range(40, 40 + BS)), list(range(70, 70 + BS))
    # two sequences admitted together: 2 computes its own copy of a0 and indexes b1 under 1's a0 block
    cm.allocate(1)
    cm.allocate(2)
    cm.prepare_inputs([1, 2], [2 * BS + 1] * 2, [], 128, 0, [], 0, a0 + a1 + [1] + a0 + b1 + [1])
    parent, _, _ = cm.block_table(1)
    child = cm.block_table(2)[1]
    assert cm.is_cached(parent) and cm.is_cached(child) and not cm.is_cached(cm.block_table(2)[0])
    assert cm.match_prefix(9, a0 + b1 + [1]) == 2 * BS
    cm.free(9)
    cm.free(1)                                                # 1's blocks become evictable, the tail free
    cm.allocate(3)
    cm.append(3, 3 * BS)                                      # the free block, then evictions: a1's, then the parent
    assert parent in cm.block_table(3) and not cm.is_cached(parent)
    assert cm.is_cached(child) and cm.match_prefix(4, a0 + b1 + [1]) == 0
    cm.free(3)
    cm.free(4)
    _fill(cm, 5, a0)                                          # the parent's block id, indexed again with a0 itself
    assert cm.block_table(5) == [parent]
    assert cm.match_prefix(6, a0 + b1 + [1]) == BS            # a0 hits again; the child chained to the evicted entry
    assert cm.is_cached(child)                                # is still indexed, and still cannot be reached


def test_randomised_admission_never_writes_shared_rows_and_failed_calls_change_nothing():
    rnd = random.Random(0)
    nb = 24
    cm = _planner.PagedKVCacheManager(nb, BS, True)
    base = [rnd.randint(3, 50) for _ in range(3 * BS)]
    live = {}                                                 # sid -> token list laid out so far (+ pending tail)
    next_id = 1
    for _ in range(400):
        op = rnd.random()
        if op < 0.25 and len(live) < 6:
            n = rnd.randint(1, 3 * BS + 8)
            toks = (base[:rnd.choice([0, BS, 2 * BS, n])] + [rnd.randint(3, 50) for _ in range(n)])[:n]
            sid, next_id = next_id, next_id + 1
            hit = cm.match_prefix(sid, toks)
            assert hit % BS == 0 and hit < len(toks) and cm.length(sid) == hit
            live[sid] = [toks, hit]
        elif op < 0.4 and live:                               # finish or preempt: both free the sequence
            sid = rnd.choice(list(live))
            cm.free(sid)
            del live[sid]
        elif live:
            pre = [s for s in live if live[s][1] < len(live[s][0])]
            dec = [s for s in live if live[s][1] >= len(live[s][0])]
            rnd.shuffle(pre)
            pre, dec = pre[:2], dec[:3]
            lens = [min(len(live[s][0]) - live[s][1], rnd.randint(1, 24)) for s in pre]
            ids = [t for s, n in zip(pre, lens) for t in live[s][0][live[s][1]:live[s][1] + n]]
            new = {s: rnd.randint(3, 50) for s in dec}
            ids += [new[s] for s in dec]
            before = {b: (cm.ref_count(b), cm.is_cached(b)) for b in range(nb)}
            free0, lengths0 = cm.num_free_blocks, {s: cm.length(s) for s in live}
            try:
                out = cm.prepare_inputs(pre, lens, dec, 128, nb * BS, [], 0, ids)
            except RuntimeError:
                assert cm.num_free_blocks == free0 and {s: cm.length(s) for s in live} == lengths0
                continue
            for t in range(out["num_tokens"]):
                b = out["slot"][t] // BS
                refs, cached = before[b]
                # a held block written to is private and unindexed; an unheld cached block may be evicted and reused
                assert refs == 0 or (refs == 1 and not cached), (t, b, before[b])
            assert out["chunk_len"] == lens and out["chunk_pos"] == [live[s][1] for s in pre]
            assert out["chunk_start"] == [sum(lens[:i]) for i in range(len(lens))]
            for s, n in zip(pre, lens):
                live[s][1] += n
            for s in dec:
                live[s][0].append(new[s])
                live[s][1] += 1
        with pytest.raises(ValueError):                       # a throwing match changes nothing
            if live:
                s = next(iter(live))
                cm.match_prefix(s, live[s][0])
            else:
                raise ValueError
        held = sum(len(cm.block_table(s)) for s in live)
        assert cm.num_free_blocks + len({b for s in live for b in cm.block_table(s)}) == nb and held >= 0


def test_caching_off_lays_out_batches_as_before():
    """Without token ids a prefix-caching manager indexes nothing, so it must hand out the blocks the plain manager
    does; and a plain manager returns no chunk descriptors."""
    rnd = random.Random(1)
    a, b = _planner.PagedKVCacheManager(20, BS), _planner.PagedKVCacheManager(20, BS, True)
    live = []
    for i in range(60):
        if rnd.random() < 0.3 or not live:
            live.append(i)
            a.allocate(i)
            b.allocate(i)
        elif rnd.random() < 0.2:
            s = live.pop(rnd.randrange(len(live)))
            a.free(s)
            b.free(s)
        pre = live[:2]
        lens = [rnd.randint(1, 9) for _ in pre]
        try:
            x = a.prepare_inputs(pre, lens, live[2:], 64, 0)
        except RuntimeError:
            with pytest.raises(RuntimeError):
                b.prepare_inputs(pre, lens, live[2:], 64, 0)
            continue
        y = b.prepare_inputs(pre, lens, live[2:], 64, 0)
        assert "chunk_len" not in x and y.pop("chunk_len") == lens
        y.pop("chunk_start"), y.pop("chunk_pos")
        assert x == y
    assert b.num_cached_blocks == 0


# ---------------------------------------------------------------------------------------------------------- reference op
def test_paged_prefill_reference_equals_ragged_reference():
    g = torch.Generator().manual_seed(0)
    bs, hkv, G, D = 16, 2, 2, 64
    nblk = 12
    slots = nblk * bs + 1
    k = torch.randn(slots, hkv, D, generator=g).bfloat16()
    v = torch.randn(slots, hkv, D, generator=g).bfloat16()
    perm = torch.randperm(nblk, generator=g).tolist()
    chunks = [(0, 5, 30), (5, 17, 0), (22, 1, 47)]            # (start, len, pos)
    table = torch.zeros(len(chunks), 4, dtype=torch.int32)
    for c, (_, n, p) in enumerate(chunks):
        for j in range(-(-(p + n) // bs)):
            table[c, j] = perm.pop()
    T = 23
    q = torch.randn(T, hkv * G, D, generator=g).bfloat16()
    cs, cl, cp = (torch.tensor([c[i] for c in chunks], dtype=torch.int32) for i in range(3))
    o = ops.paged_prefill_attention(q, k, v, table, bs, cs, cl, cp, 0.125)
    seq = torch.tensor([c for c, (_, n, _) in enumerate(chunks) for _ in range(n)], dtype=torch.int32)
    ctx = torch.tensor([p + i + 1 for _, n, p in chunks for i in range(n)], dtype=torch.int32)
    want = ops.ragged_attention(q, k, v, seq, ctx, 0.125, 64, None, table, bs)
    assert torch.allclose(o.float(), want.float(), atol=1e-2, rtol=0)
    with pytest.raises(ValueError):                           # a table row too short for its chunk
        ops.paged_prefill_attention(q, k, v, table[:, :2], bs, cs, cl, cp, 0.125)


# --------------------------------------------------------------------------------------------------- pool and model
def tiny(arch="opt", **kw):
    base = dict(arch=arch, vocab_size=96, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, ffn_dim=128,
                max_position_embeddings=256, dtype=torch.float32)
    base.update(kw)
    return OPTConfig(**base)


def _model(arch):
    kw = {"num_key_value_heads": 2} if arch == "llama" else {}
    return DecoderLM(tiny(arch, **kw), device="cpu", seed=3)


def _prompts(seed, n=6, preamble=32, lo=8, hi=48, V=96):
    rnd = random.Random(seed)
    pre = [rnd.randint(3, V - 1) for _ in range(preamble)]
    return [pre + [rnd.randint(3, V - 1) for _ in range(rnd.randint(lo, hi))] for _ in range(n)]


def _cfg(caching, **kw):
    base = dict(batch_size=128, cache_size=512, max_cache_per_seq=128, kv_block_size=BS, prefix_caching=caching)
    base.update(kw)
    return InputPoolConfig(**base)


def _logits_by_step(m, cfg, waves, new_tokens=5):
    """{(sequence id, generated count): logits} of a run whose sampler forces a fixed token per (sequence, step);
    each wave of prompts enters once the previous wave has finished its prefills."""
    gen = SequenceGenerator(m, cfg)
    pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                   max_new_tokens=new_tokens)
    seen = {}

    def forced(logits):
        rows = pool._current
        for r, p in enumerate(rows):
            seen[(p.sentence_id, p.generation_length)] = logits[r].clone()
        return torch.tensor([3 + (7 * p.sentence_id + 5 * p.generation_length) % 90 for p in rows])
    for wave in waves:
        pool.enter_prompts(wave)
        gen.step(pool, forced)
        while pool.todo:
            gen.step(pool, forced)
    while not pool.is_finished():
        gen.step(pool, forced)
    return seen, pool


@pytest.mark.parametrize("arch", ["opt", "llama"])
def test_generation_with_caching_equals_caching_off(arch):
    m = _model(arch)
    prompts = _prompts(7)
    prompts += [prompts[0], prompts[0]]                       # identical prompts
    want = SequenceGenerator(m, _cfg(False)).generate(prompts, max_new_tokens=10)
    for cfg in [_cfg(True), _cfg(True, cache_size=192, batch_size=64)]:   # roomy; tight: preemptions
        gen = SequenceGenerator(m, cfg)
        pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                       max_new_tokens=10)
        pool.enter_prompts(prompts[:2])
        gen.step(pool)
        pool.enter_prompts(prompts[2:])                       # later arrivals hit the shared preamble
        while not pool.is_finished():
            gen.step(pool)
        assert pool.get_results() == want
        assert pool.prefix_hit_tokens > 0


@pytest.mark.parametrize("arch", ["opt", "llama"])
def test_logits_with_caching_equal_caching_off(arch):
    m = _model(arch)
    prompts = _prompts(11, n=5)
    waves = [prompts[:1], prompts[1:3], prompts[3:] + [prompts[0]]]
    want, _ = _logits_by_step(m, _cfg(False), waves, 12)
    for cfg, what in [(_cfg(True), "roomy"), (_cfg(True, cache_size=96, batch_size=48), "tight")]:
        got, pool = _logits_by_step(m, cfg, waves, 12)
        assert got.keys() == want.keys(), what
        assert pool.prefix_hit_tokens > 0, what
        if what == "tight":
            assert pool.num_preemptions > 0
        scale = max(float(v.abs().max()) for v in want.values())
        err = max(float((got[k] - want[k]).abs().max()) for k in want)
        assert err <= 1e-4 * max(1.0, scale), (what, err, scale)


def test_hit_tokens_of_a_scripted_arrival_order():
    m = _model("llama")
    pre = list(range(3, 3 + 2 * BS))                          # a 32-token preamble: two full blocks
    a, b, c = pre + [50] * 10, pre + [60] * 20, pre + [70] * 5
    gen = SequenceGenerator(m, _cfg(True))
    pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                   max_new_tokens=8)
    pool.enter_prompts([a])
    gen.step(pool)                                            # a prefills 42 tokens: blocks 0 and 1 are indexed
    assert pool.prefix_hit_tokens == 0 and pool.prefill_tokens_computed == 42
    pool.enter_prompts([b, c, pre])                           # 32 + 32 hit; `pre` alone: capped at 16
    gen.step(pool)
    assert pool.prefix_hit_tokens == 32 + 32 + 16
    assert pool.prefill_tokens_computed == 42 + 20 + 5 + 16
    while not pool.is_finished():
        gen.step(pool)
    assert pool.cache_manager.num_sequences == 0 and pool.cache_manager.num_free_blocks == 512 // BS


def test_preempted_sequence_recomputes_only_its_tail():
    # two 36-token prompts in 6 blocks: at 48 tokens both need a fourth block, so the later one is preempted.  Its
    # blocks are released last one first, the running sequence's next block evicts only that tail, and the victim
    # comes back with its first two blocks from the cache.
    pool = IterationLevelInputPool(_cfg(True, cache_size=6 * BS), max_new_tokens=20)
    pool.enter_prompts([[5] * (2 * BS + 4), [6] * (2 * BS + 4)])
    cm = pool.cache_manager
    while pool.num_preemptions == 0:
        bt = pool.next()
        pool.update([7] * len(bt["logit_index"]))
    victim = pool.todo[0]
    assert victim.filled == 0 and len(victim.fill_ids) == 3 * BS + 1     # prompt + 13 generated
    hits, computed = pool.prefix_hit_tokens, pool.prefill_tokens_computed
    while not cm.has(victim.sentence_id):
        bt = pool.next()
        pool.update([7] * len(bt["logit_index"]))
    assert pool.prefix_hit_tokens - hits == 2 * BS and victim.filled == 2 * BS
    while not pool.is_finished():
        bt = pool.next()
        pool.update([7] * len(bt["logit_index"]))
    assert pool.prefill_tokens_computed - computed == BS + 1  # only the evicted block and the pending token
    assert [len(r) for r in pool.get_results()] == [2 * BS + 24] * 2


def test_config_errors():
    with pytest.raises(ValueError, match="kv_block_size"):
        IterationLevelInputPool(InputPoolConfig(cache_size=64, kv_block_size=8, prefix_caching=True))
    with pytest.raises(ValueError, match="paged"):
        IterationLevelInputPool(InputPoolConfig(prefix_caching=True))
    bloom = DecoderLM(tiny("bloom"), device="cpu", seed=0)
    with pytest.raises(ValueError, match="ALiBi"):
        SequenceGenerator(bloom, _cfg(True))
    fp8 = DecoderLM(tiny("opt", kv_cache_dtype="fp8"), device="cpu", seed=0)
    with pytest.raises(ValueError, match="fp8"):
        SequenceGenerator(fp8, _cfg(True))
    with pytest.raises(ValueError, match="kv_block_size"):
        SequenceGenerator(_model("opt"), InputPoolConfig(cache_size=64, kv_block_size=8, prefix_caching=True))


def test_model_worker_reuses_across_requests_and_starts_clean_after_a_failure():
    from alpa_b200.serve.model_worker import LangModelWorker
    m = _model("llama")
    prompts = _prompts(3, n=3)

    async def serve(w, ps):
        res = await asyncio.wait_for(asyncio.gather(*[w.completions(p, 6) for p in ps]), 120)
        return [r["ids"] for r in res]

    async def run():
        plain = LangModelWorker(m, _cfg(False))
        want = await serve(plain, prompts)
        await plain.shutdown()
        w = LangModelWorker(m, _cfg(True))
        got = await serve(w, prompts[:1]) + await serve(w, prompts[1:])
        hits = w.pool.prefix_hit_tokens                   # the long-lived pool matched the earlier request's blocks
        real = w.engine.step

        def boom(*a, **k):                                # one failing iteration after the K/V of a prompt is indexed
            real(*a, **k)
            w.engine.step = real
            raise RuntimeError("injected")
        w.engine.step = boom
        with pytest.raises(RuntimeError):
            await serve(w, prompts[:1])
        fresh = w.pool.cache_manager.num_cached_blocks, w.pool.prefix_hit_tokens
        again = await serve(w, prompts)
        await w.shutdown()
        return want, got, hits, fresh, again
    want, got, hits, fresh, again = asyncio.run(run())
    assert got == want and hits > 0
    assert fresh == (0, 0)                                # the new pool starts with an empty index
    assert again == want
