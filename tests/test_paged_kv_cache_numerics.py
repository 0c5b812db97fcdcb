"""The paged ragged attention kernel on the GPU: against float64 `ragged_ref` on the keys gathered through the block
table, bit for bit against the contiguous kernel (on a gathered copy and under an identity table), and whole serving
iterations in paged mode against contiguous mode.

Blocks are shuffled and interleaved between sequences.  Every cache row no sequence owns (free blocks, the unused rows
of each sequence's last block, the scratch row) is NaN, so a wrong row shows up in the output; padding tokens must be
exactly zero and the cache must be unchanged by the call.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, Checker, _bf, _report  # noqa: E402
from test_serving_attention_numerics import RAGGED_DIMS, ragged_ref  # noqa: E402

pytestmark = pytest.mark.gpu

NAN = float("nan")
E4M3_NAN = 0x7F
H, HKV = 8, 2                                     # grouped-query attention, group 4
# (sequence length, query tokens): a prompt chunk, decode tokens, a one-key sequence and a 16 000-key token whose
# score buffer takes the > 48 KB dynamic shared memory path
CHUNKS = [(129, 3), (1, 1), (300, 2), (40, 40), (16000, 1)]


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


def _poisoned(slots, D, fp8):
    from alpa_b200 import ops
    if not fp8:
        return torch.full((slots, HKV, D), NAN, device="cuda", dtype=BF16)
    c = ops.Fp8KV.zeros((slots, HKV, D), "cuda")
    c.data.view(torch.uint8).fill_(E4M3_NAN)
    c.scale.fill_(NAN)
    return c


def _fill(c, rows, gen):
    """Random rows (quantised by the reference quantiser for fp8) at cache rows `rows`."""
    from alpa_b200.ops import primitives as P
    x = (torch.randn(len(rows), HKV, c.shape[-1] if isinstance(c, torch.Tensor) else c.data.shape[-1],
                     generator=gen, device="cuda") * 2).to(BF16)
    if isinstance(c, torch.Tensor):
        c[rows] = x
    else:
        q, s = P._kv_quant_ref(x.cpu())
        c.data.view(torch.uint8)[rows] = q.view(torch.uint8).cuda()
        c.scale[:, rows] = s.t().cuda()


def _gather(c, rows):
    from alpa_b200 import ops
    if isinstance(c, torch.Tensor):
        return c[rows].clone()
    return ops.Fp8KV(c.data.view(torch.uint8)[rows].view(torch.float8_e4m3fn).clone(), c.scale[:, rows].clone())


def _values64(c):
    if isinstance(c, torch.Tensor):
        return c.to(F64)
    return c.data.to(F64) * c.scale.t()[..., None].to(F64)


def _bits(c):
    if isinstance(c, torch.Tensor):
        return [c.view(torch.int16).clone()]
    return [c.data.view(torch.uint8).clone(), c.scale.view(torch.int32).clone()]


def _paged_batch(D, bs, fp8, seed):
    """(q, paged k / v, table, seq_start rows, ctx_len, gathered contiguous k / v, their seq_start, max_ctx)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    nb = [-(-n // bs) for n, _ in CHUNKS]
    nblk = sum(nb) + 3                             # three blocks nobody owns
    slots = nblk * bs + 1                          # + the scratch row
    perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed)).tolist()
    blocks = [[] for _ in CHUNKS]
    for r in range(max(nb)):                       # interleave: round-robin over the sequences
        for i, b in enumerate(blocks):
            if r < nb[i]:
                b.append(perm.pop())
    mc = max(n for n, _ in CHUNKS)
    width = -(-mc // bs) + 1
    kc, vc = _poisoned(slots, D, fp8), _poisoned(slots, D, fp8)
    rows, starts, ss, sc, cl = [], [], [], [], []
    for i, (n, k) in enumerate(CHUNKS):
        starts.append(len(rows))
        rows += [blocks[i][j // bs] * bs + j % bs for j in range(n)]
        for j in range(n - k, n):
            ss.append(i)
            sc.append(starts[i])
            cl.append(j + 1)
    ss += [0, 0]
    sc += [0, 0]
    cl += [0, 0]
    rows_t = torch.tensor(rows, device="cuda")
    _fill(kc, rows_t, gen)
    _fill(vc, rows_t, gen)
    table = torch.tensor([b + [0] * (width - len(b)) for b in blocks], dtype=torch.int32, device="cuda")
    q = torch.randn(len(cl), H, D, generator=gen, device="cuda").to(BF16)
    gk, gv = _gather(kc, rows_t), _gather(vc, rows_t)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    return q, kc, vc, table, i32(ss), i32(cl), gk, gv, i32(sc), mc


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("bs", [1, 16, 64, 256])
@pytest.mark.parametrize("D", RAGGED_DIMS)
def test_paged_kernel(C, D, bs, fp8):
    from alpa_b200.ops import primitives as P
    ck = Checker()
    alibi = torch.tensor([2.0 ** (-8 * (i + 1) / H) for i in range(H)], device="cuda")
    q, kc, vc, table, ss, cl, gk, gv, sc, mc = _paged_batch(D, bs, fp8, 1000 * D + bs + fp8)
    before = _bits(kc) + _bits(vc)
    G = H // HKV
    k64, v64 = (_values64(x).repeat_interleave(G, 1) for x in (gk, gv))
    for ab in (None, alibi):
        name = f"paged D{D} bs{bs} {'fp8' if fp8 else 'bf16'}{' alibi' if ab is not None else ''}"
        got = P.ragged_attention(q, kc, vc, ss, cl, D ** -0.5, mc, ab, table, bs)
        ref = ragged_ref(q, k64, v64, sc.cpu(), cl.cpu(), D ** -0.5, ab)
        ck.bf16(f"paged ragged_attention D{D}", name, got, ref, _bf(ref))
        ck.require(bool((got[cl == 0] == 0).all()), f"{name}: padding tokens are not exactly zero")
        contiguous = P.ragged_attention(q, gk, gv, sc, cl, D ** -0.5, mc, ab)
        ck.require(torch.equal(got.view(torch.int16), contiguous.view(torch.int16)),
                   f"{name}: differs from the contiguous kernel on the gathered cache")
    after = _bits(kc) + _bits(vc)
    ck.require(all(torch.equal(a, b) for a, b in zip(before, after)), f"paged D{D} bs{bs}: the cache changed")
    assert not P.library_fallbacks()
    _report(ck)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_identity_table_equals_contiguous(C, fp8):
    """Sequences in block-aligned ranges of one cache: the contiguous kernel with seq_start = first row and the paged
    kernel with the table of consecutive blocks read the same rows and give the same bits."""
    from alpa_b200.ops import primitives as P
    D, bs = 128, 16
    gen = torch.Generator(device="cuda").manual_seed(7)
    lens = [(70, 3), (1, 1), (4000, 1), (33, 33)]
    nb = [-(-n // bs) for n, _ in lens]
    slots = sum(nb) * bs + 1
    kc, vc = _poisoned(slots, D, fp8), _poisoned(slots, D, fp8)
    table, ss, sc, cl, b0 = [], [], [], [], 0
    width = max(nb)
    for i, (n, k) in enumerate(lens):
        rows = torch.arange(b0 * bs, b0 * bs + n, device="cuda")
        _fill(kc, rows, gen)
        _fill(vc, rows, gen)
        table.append(list(range(b0, b0 + nb[i])) + [0] * (width - nb[i]))
        for j in range(n - k, n):
            ss.append(i)
            sc.append(b0 * bs)
            cl.append(j + 1)
        b0 += nb[i]
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device="cuda")  # noqa: E731
    q = torch.randn(len(cl), H, D, generator=gen, device="cuda").to(BF16)
    mc = max(n for n, _ in lens)
    got = P.ragged_attention(q, kc, vc, i32(ss), i32(cl), D ** -0.5, mc, None, i32(table), bs)
    want = P.ragged_attention(q, kc, vc, i32(sc), i32(cl), D ** -0.5, mc)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    assert not P.library_fallbacks()


def test_binding_rejects_bad_tables(C):
    from alpa_b200.ops import primitives as P
    q, kc, vc, table, ss, cl, *_, mc = _paged_batch(64, 16, False, 3)
    with pytest.raises(RuntimeError):
        P.ragged_attention(q, kc, vc, ss, cl, 0.125, mc, None, table, 24)          # not a power of two
    with pytest.raises(RuntimeError):
        P.ragged_attention(q, kc, vc, ss, cl, 0.125, mc, None, table[:, :-2], 16)  # too few blocks for max_ctx
    with pytest.raises(RuntimeError):
        P.ragged_attention(q, kc, vc, ss, cl, 0.125, mc, None, table.long(), 16)


# ------------------------------------------------------------------------------------------------------- forward pass
def _model(arch, cache):
    from alpa_b200.model.opt_model import DecoderLM, OPTConfig
    if arch == "llama":
        cfg = OPTConfig(arch="llama", vocab_size=512, hidden_size=512, num_hidden_layers=2, num_attention_heads=8,
                        num_key_value_heads=2, ffn_dim=1024, kv_cache_dtype=cache)
    else:
        cfg = OPTConfig(vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, ffn_dim=1024,
                        max_position_embeddings=512, dtype=torch.bfloat16, kv_cache_dtype=cache)
    return DecoderLM(cfg, device="cuda", seed=2)


@pytest.mark.parametrize("cache", ["bf16", "fp8"])
@pytest.mark.parametrize("arch", ["opt", "llama"])
def test_paged_iterations_have_bitwise_equal_logits(C, arch, cache):
    """Both modes admit every prompt in the first iteration (the cache is large enough), so every iteration has the
    same tokens in the same order; only the cache rows differ, and the logits must be the same bits."""
    from alpa_b200.ops import primitives as P
    from alpa_b200.serve.batching import InputPoolConfig, IterationLevelInputPool, SequenceGenerator
    m = _model(arch, cache)
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(3, 512, (int(n),), generator=g).tolist() for n in (5, 90, 17, 200, 1, 64)]
    runs = {}
    for bs in (None, 16):
        gen = SequenceGenerator(m, InputPoolConfig(batch_size=512, cache_size=2048, max_cache_per_seq=320,
                                                   kv_block_size=bs))
        pool = IterationLevelInputPool(gen.pool_config, pad_token_id=m.cfg.pad_token_id, eos_token_id=-1,
                                       max_new_tokens=24)
        pool.enter_prompts(prompts)
        seen = []

        def record(logits):
            seen.append(logits.clone())
            return logits.argmax(-1)
        while not pool.is_finished():
            gen.step(pool, record)
        runs[bs] = (seen, pool.get_results())
    (lc, rc), (lp, rp) = runs[None], runs[16]
    assert rc == rp and len(lc) == len(lp) == 24
    for i, (a, b) in enumerate(zip(lc, lp)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"iteration {i}: logits differ"
    # the tiny OPT head's GEMM (a few logit rows) may fall back in both modes; the attention must not
    assert not [f for f in P.library_fallbacks() if f[0] == "ragged_attention"]
