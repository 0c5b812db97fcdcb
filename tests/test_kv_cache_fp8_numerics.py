"""The fp8 KV-cache kernels on the GPU: the quantising store, the dequantising load, the decode kernel over an fp8
cache (append, untouched rows, accuracy, graph replay), the ragged kernel, the dispatch of every new or extended op,
and Llama / OPT decoders generating through the captured decode graph with an fp8 cache.

The cache format is `ops.Fp8KV`: e4m3 rows q with one fp32 scale s per (token, K/V head), value float(q) * s.  Bytes the
kernels write must equal the reference quantiser (`primitives._kv_quant_ref`, run on the CPU) bit for bit.  Attention
outputs are checked with `bf16_rule` against float64 references computed from the cache's values in float64.  Rows at
or past the valid length are poisoned (data 0x7F, the e4m3 NaN, and NaN scales): a kernel that reads them returns NaN,
and every byte other than the appended row must be unchanged."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, Checker, _bf, _report, bf16_rule  # noqa: E402
from test_llama_serving_numerics import DECODE_CASES, _lengths, _splits  # noqa: E402
from test_native_dispatch import _assert_same, _bits, _reference  # noqa: E402

from alpa_b200 import ops  # noqa: E402
from alpa_b200.ops import primitives as P  # noqa: E402

pytestmark = pytest.mark.gpu

NAN = float("nan")
E4M3_NAN = 0x7F


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    assert ops.native_available()
    return ops.native_module()


@pytest.fixture(autouse=True)
def _own_fallback_record(monkeypatch):
    monkeypatch.setattr(P, "_FALLBACK_SEEN", set())


def _quant_cpu(x):
    """(q as uint8, s) of bf16 rows x [..., D] by the reference quantiser on the CPU, moved to x's device."""
    q, s = P._kv_quant_ref(x.cpu())
    return q.view(torch.uint8).to(x.device), s.to(x.device)


def _filled(shape, n):
    """An Fp8KV of data shape [B, S, H, D] whose rows [0, n) hold quantised randn rows and whose other rows are
    poisoned."""
    B, S, H, D = shape
    c = ops.Fp8KV.zeros(shape, "cuda")
    c.data.view(torch.uint8).fill_(E4M3_NAN)
    c.scale.fill_(NAN)
    if n > 0:
        q, s = _quant_cpu((torch.randn(B, n, H, D, device="cuda") * 3).to(BF16))
        c.data.view(torch.uint8)[:, :n] = q
        c.scale[:, :, :n] = s.transpose(1, 2)
    return c


def _snapshot(c):
    return c.data.view(torch.uint8).clone(), c.scale.clone()


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ----------------------------------------------------------------------------------------------------------- store / load
@pytest.mark.parametrize("D", [64, 80, 128])
def test_store_kernel_prefill_rows(C, D):
    torch.manual_seed(D)
    B, T, Hkv, G, S, start = 3, 37, 2, 4, 100, 21
    qkv = (torch.randn(B, T, Hkv, G + 2, D, device="cuda") * 2).to(BF16)
    qkv[0, 3, 1, G] *= 1e4                                   # a row with a large amax
    qkv[1, 5, 0, G + 1] = 0                                  # a zero row
    k, v = qkv[:, :, :, G], qkv[:, :, :, G + 1]              # strided views of the packed projection
    kc, vc = _filled((B, S, Hkv, D), 0), _filled((B, S, Hkv, D), 0)
    k0, v0 = _snapshot(kc), _snapshot(vc)
    ops.kv_cache_store(k, v, kc, vc, start)
    assert not P.library_fallbacks()
    for c, x, (d0, s0) in ((kc, k, k0), (vc, v, v0)):
        q, s = _quant_cpu(x)
        d_want, s_want = d0.clone(), s0.clone()
        d_want[:, start:start + T] = q
        s_want[:, :, start:start + T] = s.transpose(1, 2)
        assert torch.equal(c.data.view(torch.uint8), d_want), "cache bytes differ from the reference quantiser"
        assert _same_bits(c.scale, s_want), "scales differ from the reference quantiser"


@pytest.mark.parametrize("D", [64, 80, 128])
def test_store_kernel_slots(C, D):
    torch.manual_seed(D + 1)
    T, Hkv, G, slots = 29, 4, 1, 300
    qkv = torch.randn(T, Hkv, G + 2, D, device="cuda").to(BF16)
    k, v = qkv[None, :, :, G], qkv[None, :, :, G + 1]
    rows = torch.randperm(slots, device="cuda")[:T]
    kc = ops.Fp8KV.zeros((slots, Hkv, D), "cuda")
    vc = ops.Fp8KV.zeros((slots, Hkv, D), "cuda")
    for c in (kc, vc):
        c.data.view(torch.uint8).fill_(E4M3_NAN)
        c.scale.fill_(NAN)
    k0, v0 = _snapshot(kc), _snapshot(vc)
    ops.kv_cache_store(k, v, kc, vc, rows=rows)
    assert not P.library_fallbacks()
    for c, x, (d0, s0) in ((kc, k, k0), (vc, v, v0)):
        q, s = _quant_cpu(x[0])
        d_want, s_want = d0.clone(), s0.clone()
        d_want[rows] = q
        s_want[:, rows] = s.t()
        assert torch.equal(c.data.view(torch.uint8), d_want)
        assert _same_bits(c.scale, s_want)


@pytest.mark.parametrize("D", [64, 80, 128])
def test_load_kernel(C, D):
    torch.manual_seed(D + 2)
    B, S, H, end = 2, 70, 3, 51
    c = _filled((B, S, H, D), end)
    out = ops.kv_cache_load(c, end)
    assert not P.library_fallbacks()
    cpu = ops.Fp8KV(c.data.cpu(), c.scale.cpu())
    assert _same_bits(out.cpu(), cpu.values(end).to(BF16))


# ----------------------------------------------------------------------------------------------------------- decode
def _decode_ref(qf, k, v, scale):
    """o [B, Hkv, G, D] float64 of queries qf [B, Hkv, G, D] over the cache values k / v [B, n, Hkv, D]."""
    s = torch.einsum("bhgd,bnhd->bhgn", qf.to(F64), k.to(F64)) * scale
    return torch.einsum("bhgn,bnhd->bhgd", torch.softmax(s, -1), v.to(F64))


def _values64(c, n):
    return c.data[:, :n].to(F64) * c.scale[:, :, :n].transpose(1, 2)[..., None].to(F64)


def _check_append(kc, vc, k0, v0, n, k_new, v_new):
    """The appended row n - 1 equals the reference quantiser of k_new / v_new [B, Hkv, D]; no other byte changed."""
    for c, x, (d0, s0) in ((kc, k_new, k0), (vc, v_new, v0)):
        q, s = _quant_cpu(x)
        d_want, s_want = d0.clone(), s0.clone()
        d_want[:, n - 1] = q
        s_want[:, :, n - 1] = s
        assert torch.equal(c.data.view(torch.uint8), d_want), "appended row / untouched rows differ"
        assert _same_bits(c.scale, s_want), "appended scale / untouched scales differ"


@pytest.mark.parametrize("rope", [False, True])
@pytest.mark.parametrize("G,Hkv,D,B", DECODE_CASES)
def test_decode_kernel_fp8(C, G, Hkv, D, B, rope):
    torch.manual_seed(G * 100 + Hkv * 10 + D + B + rope)
    S_max, theta = 160, 500000.0
    scale = D ** -0.5
    splits = _splits(B, Hkv, G)
    ck = Checker()
    for n in _lengths(S_max, min(splits, 10)):
        pos = torch.randint(n - 1, 100000, (B, 1), device="cuda") if rope else None
        qkv = (torch.randn(B, 1, Hkv, G + 2, D, device="cuda") * 2).to(BF16)
        kc, vc = _filled((B, S_max, Hkv, D), n - 1), _filled((B, S_max, Hkv, D), n - 1)
        k0, v0 = _snapshot(kc), _snapshot(vc)
        rot = ops.rotary_packed(qkv, pos, theta, False)[:, 0] if rope else qkv[:, 0]
        o = ops.fast.decode_attention_gqa(qkv, kc, vc, torch.tensor([n], dtype=torch.int32, device="cuda"), pos,
                                          scale, theta)
        _check_append(kc, vc, k0, v0, n, rot[:, :, G], qkv[:, 0, :, G + 1])
        ref = _decode_ref(rot[:, :, :G], _values64(kc, n), _values64(vc, n), scale)
        ck._add(("decode_fp8", "fwd"), bf16_rule(f"G={G} Hkv={Hkv} D={D} B={B} rope={rope} n={n}",
                                                 o.view(B, Hkv, G, D), ref, _bf(ref)))
    assert not P.library_fallbacks()
    _report(ck)


def test_decode_multi_head_binding_fp8(C):
    """decode_attention (separate q / k_new / v_new views, the OPT decode path) over an fp8 cache."""
    torch.manual_seed(3)
    B, h, D, S_max, n = 3, 12, 64, 300, 211
    qkv = torch.randn(B, 1, h, 3, D, device="cuda").to(BF16)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    kc, vc = _filled((B, S_max, h, D), n - 1), _filled((B, S_max, h, D), n - 1)
    k0, v0 = _snapshot(kc), _snapshot(vc)
    o = ops.fast.decode_attention(q, k, v, kc, vc, torch.tensor([n], dtype=torch.int32, device="cuda"), D ** -0.5)
    _check_append(kc, vc, k0, v0, n, k[:, 0], v[:, 0])
    ref = _decode_ref(q[:, 0, :, None], _values64(kc, n), _values64(vc, n), D ** -0.5)
    ck = Checker()
    ck._add(("decode_fp8", "mha"), bf16_rule("mha", o.view(B, h, 1, D), ref, _bf(ref)))
    assert not P.library_fallbacks()
    _report(ck)


def test_decode_fp8_graph_replay(C):
    torch.manual_seed(0)
    B, Hkv, G, D, S_max, theta = 2, 8, 4, 128, 4096, 500000.0
    qkv = torch.randn(B, 1, Hkv, G + 2, D, device="cuda").to(BF16)
    kc, vc = _filled((B, S_max, Hkv, D), S_max), _filled((B, S_max, Hkv, D), S_max)
    kv_len = torch.ones(1, dtype=torch.int32, device="cuda")
    pos = torch.zeros(B, 1, dtype=torch.long, device="cuda")
    ops.fast.decode_attention_gqa(qkv, kc, vc, kv_len, pos, D ** -0.5, theta)        # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.fast.decode_attention_gqa(qkv, kc, vc, kv_len, pos, D ** -0.5, theta)
    ck = Checker()
    for n in (1, 33, 1000, 4096):
        k0, v0 = _snapshot(kc), _snapshot(vc)
        kv_len.fill_(n)
        pos.fill_(n - 1)
        g.replay()
        torch.cuda.synchronize()
        rot = ops.rotary_packed(qkv, pos, theta, False)[:, 0]
        _check_append(kc, vc, k0, v0, n, rot[:, :, G], qkv[:, 0, :, G + 1])
        ref = _decode_ref(rot[:, :, :G], _values64(kc, n), _values64(vc, n), D ** -0.5)
        ck._add(("decode_fp8", "graph"), bf16_rule(f"graph n={n}", out.view(B, Hkv, G, D), ref, _bf(ref)))
    _report(ck)


# ----------------------------------------------------------------------------------------------------------- ragged
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("G", [1, 2, 4])
def test_ragged_fp8(C, G, alibi):
    torch.manual_seed(G + 10 * alibi)
    Hkv, D, slots = 2, 128, 400
    h = Hkv * G
    lens = [37, 1, 150, 64]
    starts = [0, 40, 60, 220]
    st, cl = [], []
    for s0, n in zip(starts, lens):
        for j in (n - 1, max(0, n - 3)):
            st.append(s0)
            cl.append(j + 1)
    T = len(st)
    q = torch.randn(T, h, D, device="cuda").to(BF16)
    kc, vc = ops.Fp8KV.zeros((slots, Hkv, D), "cuda"), ops.Fp8KV.zeros((slots, Hkv, D), "cuda")
    for c in (kc, vc):
        c.data.view(torch.uint8).fill_(E4M3_NAN)
        c.scale.fill_(NAN)
        for s0, n in zip(starts, lens):
            qq, s = _quant_cpu((torch.randn(n, Hkv, D, device="cuda") * 3).to(BF16))
            c.data.view(torch.uint8)[s0:s0 + n] = qq
            c.scale[:, s0:s0 + n] = s.t()
    slopes = (torch.rand(h, device="cuda") * 0.1) if alibi else None
    st_t = torch.tensor(st, dtype=torch.int32, device="cuda")
    cl_t = torch.tensor(cl, dtype=torch.int32, device="cuda")
    o = ops.fast.ragged_attention(q, kc, vc, st_t, cl_t, D ** -0.5, 256, slopes)
    assert not P.library_fallbacks()
    kv64 = [c.data.to(F64) * c.scale.t()[..., None].to(F64) for c in (kc, vc)]
    ck = Checker()
    for t in range(T):
        n, s0 = cl[t], st[t]
        k = kv64[0][s0:s0 + n].repeat_interleave(G, 1)
        vv = kv64[1][s0:s0 + n].repeat_interleave(G, 1)
        s = torch.einsum("hd,nhd->hn", q[t].to(F64), k) * D ** -0.5
        if alibi:
            s = s + slopes.to(F64)[:, None] * torch.arange(n, dtype=F64, device="cuda")[None]
        ref = torch.einsum("hn,nhd->hd", torch.softmax(s, -1), vv)
        ck._add(("ragged_fp8", "fwd"), bf16_rule(f"t={t} G={G} alibi={alibi}", o[t], ref, _bf(ref)))
    _report(ck)


# ----------------------------------------------------------------------------------------------------------- dispatch
def _caches(shape, n=None):
    B, S = shape[:2]
    return _filled(shape, S if n is None else n), _filled(shape, S if n is None else n)


def _out(o, *caches):
    return [o] + [t for c in caches for t in (c.data.view(torch.uint8), c.scale)]


def _store(D, prefill=True):
    torch.manual_seed(D)
    qkv = torch.randn(2, 5, 3, 3, D, device="cuda").to(BF16)
    k, v = qkv[:, :, :, 1], qkv[:, :, :, 2]
    if prefill:
        def run():
            kc, vc = ops.Fp8KV.zeros((2, 9, 3, D), "cuda"), ops.Fp8KV.zeros((2, 9, 3, D), "cuda")
            ops.kv_cache_store(k, v, kc, vc, 2)
            return _out(torch.zeros(1), kc, vc)
        return run
    rows = torch.tensor([7, 1, 3, 0, 12], device="cuda")

    def run_slots():
        kc, vc = ops.Fp8KV.zeros((14, 3, D), "cuda"), ops.Fp8KV.zeros((14, 3, D), "cuda")
        ops.kv_cache_store(k[:1], v[:1], kc, vc, rows=rows)
        return _out(torch.zeros(1), kc, vc)
    return run_slots


def _load(D):
    torch.manual_seed(D)
    c = _filled((2, 9, 3, D), 9)
    return lambda: ops.kv_cache_load(c, 6)


def _decode(D):
    torch.manual_seed(D)
    qkv = torch.randn(2, 1, 3, 3, D, device="cuda").to(BF16)

    def run():
        kc, vc = _caches((2, 20, 3, D), 11)
        n = torch.tensor([12], dtype=torch.int32, device="cuda")
        return _out(ops.decode_attention(qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], kc, vc, n, 0.3), kc, vc)
    return run


def _decode_gqa(D):
    torch.manual_seed(D)
    qkv = torch.randn(2, 1, 2, 4, D, device="cuda").to(BF16)
    pos = torch.full((2, 1), 11, device="cuda")

    def run():
        kc, vc = _caches((2, 20, 2, D), 11)
        n = torch.tensor([12], dtype=torch.int32, device="cuda")
        return _out(ops.decode_attention_gqa(qkv, kc, vc, n, pos, 0.3, 10000.0), kc, vc)
    return run


def _ragged(D):
    torch.manual_seed(D)
    q = torch.randn(3, 4, D, device="cuda").to(BF16)
    kc, vc = (ops.Fp8KV(c.data[0], c.scale[0]) for c in _caches((1, 20, 2, D)))
    st = torch.tensor([0, 0, 10], dtype=torch.int32, device="cuda")
    cl = torch.tensor([5, 9, 10], dtype=torch.int32, device="cuda")
    return lambda: ops.ragged_attention(q, kc, vc, st, cl, 0.3, 16)


SUPPORTED = {
    "kv_cache_store": lambda: _store(64), "kv_cache_store_slots": lambda: _store(80, prefill=False),
    "kv_cache_load": lambda: _load(64), "decode_attention": lambda: _decode(64),
    "decode_attention_gqa": lambda: _decode_gqa(64), "ragged_attention": lambda: _ragged(64),
}
UNSUPPORTED = {
    "kv_cache_store": ("kv_cache_store", lambda: _store(12)),
    "kv_cache_store_slots": ("kv_cache_store", lambda: _store(264, prefill=False)),
    "kv_cache_load": ("kv_cache_load", lambda: _load(12)),
    "decode_attention": ("decode_attention", lambda: _decode(136)),
    "decode_attention_gqa": ("decode_attention_gqa", lambda: _decode_gqa(144)),
    "ragged_attention": ("ragged_attention", lambda: _ragged(12)),
}


@pytest.mark.parametrize("name", sorted(SUPPORTED))
def test_supported_call_launches_a_kernel(C, name):
    run = SUPPORTED[name]()
    n0 = C.launch_count()
    run()
    torch.cuda.synchronize()
    assert C.launch_count() > n0, f"{name}: no sm_90a kernel launched"
    assert P.library_fallbacks() == [], P.library_fallbacks()


@pytest.mark.parametrize("name", sorted(UNSUPPORTED))
def test_unsupported_layout_records_one_fallback(C, name):
    op, build = UNSUPPORTED[name]
    got = _bits(build()())
    torch.cuda.synchronize()
    recorded = P.library_fallbacks()
    assert len(recorded) == 1 and recorded[0][0] == op, recorded
    _assert_same(got, _reference(build), name)


@pytest.mark.parametrize("name", sorted(SUPPORTED))
def test_missing_extension_raises_unless_fallback_allowed(C, name, monkeypatch):
    build = SUPPORTED[name]
    want = _reference(build)
    monkeypatch.setattr(ops, "native_available", lambda: False)
    monkeypatch.delenv("ALPA_B200_ALLOW_FALLBACK", raising=False)
    with pytest.raises(RuntimeError, match="extension is not built"):
        build()()
    monkeypatch.setenv("ALPA_B200_ALLOW_FALLBACK", "1")
    _assert_same(_bits(build()()), want, name)


# ----------------------------------------------------------------------------------------------------------- end to end
def _decoder(arch):
    from alpa_b200.model.opt_model import DecoderLM, OPTConfig
    kw = {"llama": dict(num_key_value_heads=2, rope_theta=500000.0, ffn_dim=1536),
          "codegen": dict(ffn_dim=4096, rotary_dim=32, activation="gelu")}.get(arch, dict(ffn_dim=4096))
    if arch == "bloom":
        kw["activation"] = "gelu"
    cfg = OPTConfig(arch=arch, vocab_size=512, hidden_size=1024, num_hidden_layers=3, num_attention_heads=8,
                    kv_cache_dtype="fp8", **kw)
    return DecoderLM(cfg, device="cuda", seed=1)


@pytest.mark.parametrize("arch", ["llama", "opt", "codegen"])
def test_decoder_generates_through_graph_with_fp8_cache(C, arch, monkeypatch):
    from alpa_b200.serve import generator as gen_mod
    m = _decoder(arch)
    B = 2 if arch == "llama" else 8               # the prefill's LM head is the GEMM there: 8 rows keep it on the kernel
    gen = gen_mod.Generator(m, B, 96)
    assert isinstance(gen.cache[0][0], ops.Fp8KV)
    seen = []
    orig = gen_mod._sample

    def record(logits, *a):
        seen.append(logits.float().clone())
        return orig(logits, *a)
    monkeypatch.setattr(gen_mod, "_sample", record)
    ids = torch.randint(4, 512, (B, 40), generator=torch.Generator().manual_seed(0))
    out = gen.generate(ids, max_new_tokens=12)
    assert gen._decode_graphs, "the decode step was not captured"
    full = gen.forward(out.sequences).float()                 # eager fp8-cache forward of the generated sequence
    for t, lg in enumerate(seen):
        ref = full[:, 40 - 1 + t]
        err = (lg - ref).abs().max()
        assert err <= 0.05 * ref.abs().max() + 0.02, (t, float(err), float(ref.abs().max()))
    # like for like: every step the graph replayed against the same step run eagerly over a cache filled the same way
    seq = out.sequences.cuda()
    cache = m.init_cache(B, 96)
    m.forward(seq[:, :40], torch.arange(40, device="cuda").repeat(B, 1), cache, 0)
    for t in range(1, len(seen)):
        p = 40 - 1 + t
        kv_len = torch.full((1,), p + 1, dtype=torch.int32, device="cuda")
        eager = m.gather_logits(m.decode_step(seq[:, p:p + 1], torch.full((B, 1), p, device="cuda"), cache,
                                              kv_len))[:, -1].float()
        err = (seen[t] - eager).abs().max()
        assert err <= 2 ** -7 * eager.abs().max(), (t, float(err), float(eager.abs().max()))
    assert not P.library_fallbacks()


@pytest.mark.parametrize("arch", ["llama", "opt", "codegen", "bloom"])
def test_ragged_generation_with_fp8_cache_runs_kernels(C, arch):
    """Unequal prompts take the ragged path (slot stores, ragged attention) with every arch's K / V layout: the
    rotated K of codegen is a fresh tensor next to a strided V view, BLOOM adds ALiBi."""
    from alpa_b200.serve.generator import Generator
    m = _decoder(arch)
    prompts = [[5 + i for i in range(n)] for n in (17, 3, 40, 9, 24, 8, 31, 12)]
    out = Generator(m, 8, 96).generate(prompts, max_new_tokens=6)
    assert out.sequences.shape[0] == len(prompts)
    for p, s in zip(prompts, out.sequences.tolist()):
        assert s[:len(p)] == p
    assert not P.library_fallbacks()
