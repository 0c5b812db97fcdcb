"""The paged prefill kernel (`ops.paged_prefill_attention`) on the GPU against a float64 reference over the keys
gathered through the block table, and whole serving runs with prefix caching on against caching off.

Blocks are shuffled and interleaved between sequences.  Every cache row no chunk may read (free blocks, the unused rows
of each sequence's last block, the scratch row) is NaN, so a wrong row, or a masked row that still reaches P V, shows up
in the output.  The cache must be unchanged by the call, and two calls must give the same bits.
"""
import os
import random
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, Checker, _bf, _report  # noqa: E402

pytestmark = pytest.mark.gpu

HKV = 2
CHUNK_LENS = (1, 63, 64, 65, 512)


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from alpa_b200 import ops
    assert ops.native_available()
    return ops.native_module()


@pytest.fixture(autouse=True)
def _own_fallback_record(monkeypatch):
    from alpa_b200.ops import primitives as P
    monkeypatch.setattr(P, "_FALLBACK_SEEN", set())


def _case(bs, D, G, seed):
    """q [T, HKV * G, D], NaN-poisoned caches with the chunks' keys filled in, the table and the descriptors: every
    (cached prefix, chunk length) pair of prefixes 0, 1, bs - 1, 3 bs, 6000 x CHUNK_LENS is one chunk, in shuffled
    order."""
    pairs = [(p, n) for p in (0, 1, bs - 1, 3 * bs, 6000) for n in CHUNK_LENS]
    random.Random(seed).shuffle(pairs)
    nb = [-(-(p + n) // bs) for p, n in pairs]
    nblk = sum(nb) + 3                                  # three blocks nobody owns
    slots = nblk * bs + 1                               # + the scratch row
    perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed)).tolist()
    blocks = [[] for _ in pairs]
    for r in range(max(nb)):                            # interleave the sequences' blocks
        for i, b in enumerate(blocks):
            if r < nb[i]:
                b.append(perm.pop())
    width = max(nb) + 1
    gen = torch.Generator(device="cuda").manual_seed(seed)
    kc = torch.full((slots, HKV, D), float("nan"), device="cuda", dtype=BF16)
    vc = torch.full_like(kc, float("nan"))
    rows = []
    for i, (p, n) in enumerate(pairs):
        r = torch.tensor([blocks[i][j // bs] * bs + j % bs for j in range(p + n)], device="cuda")
        rows.append(r)
        kc[r] = (torch.randn(len(r), HKV, D, generator=gen, device="cuda") * 2).to(BF16)
        vc[r] = torch.randn(len(r), HKV, D, generator=gen, device="cuda").to(BF16)
    table = torch.tensor([b + [0] * (width - len(b)) for b in blocks], dtype=torch.int32, device="cuda")
    lens = [n for _, n in pairs]
    starts = [sum(lens[:i]) for i in range(len(lens))]
    q = (torch.randn(sum(lens), HKV * G, D, generator=gen, device="cuda") * 2).to(BF16)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    return q, kc, vc, table, i32(starts), i32(lens), i32([p for p, _ in pairs]), rows, pairs


def _ref(q, kc, vc, rows, starts, pairs, scale):
    G = q.shape[1] // HKV
    out = torch.empty(q.shape, dtype=F64, device=q.device)
    for r, s0, (p, n) in zip(rows, starts, pairs):
        k = kc[r].to(F64).repeat_interleave(G, 1)                                 # [keys, H, D]
        v = vc[r].to(F64).repeat_interleave(G, 1)
        s = torch.einsum("ihd,jhd->hij", q[s0:s0 + n].to(F64) * scale, k)
        j = torch.arange(p + n, device=q.device)
        s = s.masked_fill(j[None, None, :] > (p + torch.arange(n, device=q.device))[None, :, None], float("-inf"))
        out[s0:s0 + n] = torch.einsum("hij,jhd->ihd", torch.softmax(s, -1), v)
    return out


@pytest.mark.parametrize("G", [1, 4, 8])
@pytest.mark.parametrize("bs", [16, 64, 256])
@pytest.mark.parametrize("D", [64, 128])
def test_paged_prefill_kernel(C, D, bs, G):
    from alpa_b200.ops import primitives as P
    ck = Checker()
    q, kc, vc, table, cs, cl, cp, rows, pairs = _case(bs, D, G, 100 * D + bs + G)
    before = [kc.view(torch.int16).clone(), vc.view(torch.int16).clone()]
    scale = D ** -0.5
    got = P.paged_prefill_attention(q, kc, vc, table, bs, cs, cl, cp, scale)
    again = P.paged_prefill_attention(q, kc, vc, table, bs, cs, cl, cp, scale)
    torch.cuda.synchronize()
    assert P.library_fallbacks() == []
    ref = _ref(q, kc, vc, rows, cs.tolist(), pairs, scale)
    name = f"paged prefill D{D} bs{bs} G{G}"
    ck.bf16(f"paged_prefill_attention D{D}", name, got, ref, _bf(ref))
    ck.require(torch.equal(got.view(torch.int16), again.view(torch.int16)), f"{name}: two calls differ")
    ck.require(torch.equal(kc.view(torch.int16), before[0]) and torch.equal(vc.view(torch.int16), before[1]),
               f"{name}: the call changed the cache")
    # the grouped view of a packed projection [T, HKV, G + 2, D] gives the same bits as the [T, H, D] copy
    packed = torch.zeros(q.shape[0], HKV, G + 2, D, device="cuda", dtype=BF16)
    packed[:, :, :G] = q.view(-1, HKV, G, D)
    view = P.paged_prefill_attention(packed[:, :, :G], kc, vc, table, bs, cs, cl, cp, scale)
    ck.require(torch.equal(view.view(torch.int16), got.view(torch.int16)), f"{name}: grouped view differs")
    _report(ck)


def test_binding_checks(C):
    from alpa_b200.ops import primitives as P
    q, kc, vc, table, cs, cl, cp, _, _ = _case(16, 64, 4, 7)
    with pytest.raises(RuntimeError, match="blocks per row"):
        P.paged_prefill_attention(q, kc, vc, table[:, :3], 16, cs, cl, cp, 0.125)
    with pytest.raises(RuntimeError, match="int32"):
        P.paged_prefill_attention(q, kc, vc, table, 16, cs.long(), cl, cp, 0.125)
    with pytest.raises(RuntimeError, match="power of two"):
        C.paged_prefill_attention(q, kc, vc, table, 24, cs, cl, cp, 0.125, 8000)


# ---------------------------------------------------------------------------------------------------------- serving
def _serve(m, cfg, waves, new_tokens):
    from alpa_b200.serve.batching import IterationLevelInputPool, SequenceGenerator
    gen = SequenceGenerator(m, cfg)
    pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=2,
                                   max_new_tokens=new_tokens)
    seen = {}

    def forced(logits):
        rows = pool._current
        for r, p in enumerate(rows):
            seen[(p.sentence_id, p.generation_length)] = logits[r].float().cpu()
        return torch.tensor([3 + (7 * p.sentence_id + 5 * p.generation_length) % 500 for p in rows],
                            device=logits.device)
    for wave in waves:
        pool.enter_prompts(wave)
        gen.step(pool, forced)
        while pool.todo:
            gen.step(pool, forced)
    while not pool.is_finished():
        gen.step(pool, forced)
    return seen, pool


@pytest.mark.parametrize("arch", ["opt", "llama"])
def test_serving_with_caching_matches_caching_off(C, arch):
    from alpa_b200.model.opt_model import DecoderLM, OPTConfig
    from alpa_b200.serve.batching import InputPoolConfig
    kw = {"num_key_value_heads": 2} if arch == "llama" else {}
    cfg = OPTConfig(arch=arch, vocab_size=512, hidden_size=512, num_hidden_layers=2, num_attention_heads=8,
                    ffn_dim=1024, max_position_embeddings=1024, dtype=BF16, **kw)
    m = DecoderLM(cfg, device="cuda", seed=5)
    rnd = random.Random(0)
    pre = [rnd.randint(3, 500) for _ in range(200)]
    prompts = [pre + [rnd.randint(3, 500) for _ in range(rnd.randint(5, 150))] for _ in range(8)]
    waves = [prompts[:2], prompts[2:5], prompts[5:] + [prompts[0]]]
    pool_cfg = dict(batch_size=512, cache_size=4096, max_cache_per_seq=512, kv_block_size=16)
    want, _ = _serve(m, InputPoolConfig(**pool_cfg), waves, 8)
    got, pool = _serve(m, InputPoolConfig(prefix_caching=True, **pool_cfg), waves, 8)
    assert got.keys() == want.keys() and pool.prefix_hit_tokens > 0
    from alpa_b200.ops import primitives as P
    assert not [f for f in P.library_fallbacks() if "attention" in f[0]]
    # budget: 8 bf16 ulps of the logits' scale (the two paths round attention outputs differently)
    scale = max(float(v.abs().max()) for v in want.values())
    budget = 8 * 2.0 ** -8 * scale
    first = [k for k in want if k[1] == 0]
    err = max(float((got[k] - want[k]).abs().max()) for k in first)
    assert err <= budget, (err, budget)
    for k, w in want.items():
        top2 = torch.topk(w, 2).values
        if float(top2[0] - top2[1]) > 2 * budget:
            assert int(got[k].argmax()) == int(w.argmax()), k
