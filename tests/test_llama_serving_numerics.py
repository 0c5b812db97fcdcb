"""The Llama serving kernels against float64 references on the GPU: the grouped-query decode kernel with fused rotary
and cache append (`decode_attention_gqa`), the grouped ragged kernel, the RMSNorm prologue of the decode GEMV, and a
bf16 Llama `DecoderLM` generating through the captured decode graph.

As in test_serving_attention_numerics.py, every reference is float64 and computed from the exact bf16 values the kernel
read, and `bf16_rule` compares the kernel's error with that of the reference rounded to bf16 once.  The query heads and
the new key the decode kernel attends with are the bf16 outputs of `rotary_packed` on the same packed row; the row it
appends must equal that output bit for bit.  Cache rows at or past the valid length and the stale row the new key
replaces are NaN, and every cache byte other than the appended row must be unchanged."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, Checker, _bf, _report, bf16_rule  # noqa: E402

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from alpa_b200 import ops
    assert ops.native_available()
    return ops.native_module()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _chunk(G):
    return 1 if G == 1 else 2 if G == 2 else 4 if G <= 4 else 8


def _splits(B, Hkv, G):
    """The binding's split count: about two CTAs per SM over the (sequence, K/V head, chunk) rows, 1 to 64."""
    rows = B * Hkv * -(-G // _chunk(G))
    return max(1, min(64, (2 * _sms() + rows - 1) // rows))


def _lengths(S_max, splits):
    """kv_len values: 1, S_max, and lengths that leave the last split with a single key."""
    out = {1, S_max, 2, 17}
    for s in range(2, splits + 1):
        for n in range(1, S_max + 1):
            per = ((n + s - 1) // s + 15) // 16 * 16
            if (s - 1) * per == n - 1:
                out.add(n)
                break
    return sorted(x for x in out if 1 <= x <= S_max)


def gqa_decode_ref(rot, k, v, scale):
    """o [B, Hkv, G, D] float64 of the rotated packed row rot [B, Hkv, G + 2, D] over k / v [B, n, Hkv, D]."""
    G = rot.shape[2] - 2
    s = torch.einsum("bhgd,bnhd->bhgn", rot[:, :, :G].to(F64), k.to(F64)) * scale
    return torch.einsum("bhgn,bnhd->bhgd", torch.softmax(s, -1), v.to(F64))


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


DECODE_CASES = [  # (G, Hkv, D, B)
    (1, 8, 128, 1), (2, 2, 64, 3), (4, 8, 128, 1), (4, 8, 128, 8), (8, 1, 80, 3), (16, 2, 64, 1), (4, 1, 80, 8),
    (8, 8, 128, 3), (16, 1, 128, 8), (2, 8, 80, 1), (1, 2, 64, 8),
]


@pytest.mark.parametrize("G,Hkv,D,B", DECODE_CASES)
def test_gqa_decode_kernel(C, G, Hkv, D, B):
    from alpa_b200 import ops
    torch.manual_seed(G * 100 + Hkv * 10 + D + B)
    S_max, theta = 160, 500000.0
    scale = D ** -0.5
    splits = _splits(B, Hkv, G)
    ck = Checker()
    for n in _lengths(S_max, min(splits, 10)):
        pos = torch.randint(n - 1, 100000, (B, 1), device="cuda")
        qkv = (torch.randn(B, 1, Hkv, G + 2, D, device="cuda") * 2).to(BF16)
        k = torch.randn(B, S_max, Hkv, D, device="cuda").to(BF16)
        v = torch.randn(B, S_max, Hkv, D, device="cuda").to(BF16)
        k[:, n - 1:], v[:, n - 1:] = NAN, NAN
        k0, v0 = k.clone(), v.clone()
        rot = ops.rotary_packed(qkv, pos, theta, False)[:, 0]
        o = ops.fast.decode_attention_gqa(qkv, k, v, torch.tensor([n], dtype=torch.int32, device="cuda"), pos, scale,
                                          theta)
        assert _bits_equal(k[:, n - 1], rot[:, :, G]), "appended key != rotary_packed's"
        assert _bits_equal(v[:, n - 1], qkv[:, 0, :, G + 1]), "appended value != v_new"
        keep = torch.ones(S_max, dtype=torch.bool, device="cuda")
        keep[n - 1] = False
        assert _bits_equal(k[:, keep], k0[:, keep]) and _bits_equal(v[:, keep], v0[:, keep])
        ref = gqa_decode_ref(rot, k[:, :n], v[:, :n], scale)
        ck._add(("decode_gqa", "fwd"), bf16_rule(f"G={G} Hkv={Hkv} D={D} B={B} n={n}", o.view(B, Hkv, G, D), ref,
                                                   _bf(ref)))
    _report(ck)


def test_gqa_decode_graph_replay(C):
    from alpa_b200 import ops
    torch.manual_seed(0)
    B, Hkv, G, D, S_max, theta = 2, 8, 4, 128, 4096, 500000.0
    qkv = torch.randn(B, 1, Hkv, G + 2, D, device="cuda").to(BF16)
    k = torch.randn(B, S_max, Hkv, D, device="cuda").to(BF16)
    v = torch.randn(B, S_max, Hkv, D, device="cuda").to(BF16)
    kv_len = torch.ones(1, dtype=torch.int32, device="cuda")
    pos = torch.zeros(B, 1, dtype=torch.long, device="cuda")
    ops.fast.decode_attention_gqa(qkv, k, v, kv_len, pos, D ** -0.5, theta)       # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.fast.decode_attention_gqa(qkv, k, v, kv_len, pos, D ** -0.5, theta)
    ck = Checker()
    for n in (1, 33, 1000, 4096):
        kv_len.fill_(n)
        pos.fill_(n - 1)
        g.replay()
        torch.cuda.synchronize()
        rot = ops.rotary_packed(qkv, pos, theta, False)[:, 0]
        assert _bits_equal(k[:, n - 1], rot[:, :, G])
        ref = gqa_decode_ref(rot, k[:, :n], v[:, :n], D ** -0.5)
        ck._add(("decode_gqa", "graph"), bf16_rule(f"graph n={n}", out.view(B, Hkv, G, D), ref, _bf(ref)))
    _report(ck)


@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("G", [2, 4])
def test_ragged_gqa(C, G, alibi):
    from alpa_b200 import ops
    torch.manual_seed(G)
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
    kc = torch.full((slots, Hkv, D), NAN, device="cuda").to(BF16)
    vc = torch.full((slots, Hkv, D), NAN, device="cuda").to(BF16)
    for s0, n in zip(starts, lens):
        kc[s0:s0 + n] = torch.randn(n, Hkv, D, device="cuda").to(BF16)
        vc[s0:s0 + n] = torch.randn(n, Hkv, D, device="cuda").to(BF16)
    slopes = (torch.rand(h, device="cuda") * 0.1) if alibi else None
    st_t = torch.tensor(st, dtype=torch.int32, device="cuda")
    cl_t = torch.tensor(cl, dtype=torch.int32, device="cuda")
    o = ops.fast.ragged_attention(q, kc, vc, st_t, cl_t, D ** -0.5, 256, slopes)
    ck = Checker()
    for t in range(T):
        n, s0 = cl[t], st[t]
        k = kc[s0:s0 + n].to(F64).repeat_interleave(G, 1)
        vv = vc[s0:s0 + n].to(F64).repeat_interleave(G, 1)
        s = torch.einsum("hd,nhd->hn", q[t].to(F64), k) * D ** -0.5
        if alibi:
            s = s + slopes.to(F64)[:, None] * torch.arange(n, dtype=F64, device="cuda")[None]
        ref = torch.einsum("hn,nhd->hd", torch.softmax(s, -1), vv)
        ck._add(("ragged_gqa", "fwd"), bf16_rule(f"t={t} G={G} alibi={alibi}", o[t], ref, _bf(ref)))
    _report(ck)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("M", [1, 3, 8])
def test_rms_gemv_prologue(C, M, fp8):
    from alpa_b200 import ops
    from alpa_b200.model.opt_model import _TPLinear
    torch.manual_seed(M + 10 * fp8)
    K, N, eps = 4096, 1024, 1e-5
    x = torch.randn(M, K, device="cuda").to(BF16)
    x[0] *= 300.0                                          # a large-magnitude row
    g = (torch.rand(K, device="cuda") + 0.5).to(BF16)
    lin = _TPLinear((torch.randn(N, K, device="cuda") * 0.02).to(BF16), None, fp8)
    y = ops.fast.linear_decode(x, lin.w, lin.scale, None, ln=ops.RMSNormArgs(g, eps))
    assert not ops.primitives.library_fallbacks()
    xf = x.to(F64)
    xn = _bf(xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * g.to(F64))
    if fp8:
        # the reference of the fused path: the un-fused RMSNorm kernel, then the same fp8 GEMV
        want = ops.fast.linear_decode(ops.fast.rms_norm(x, g, eps)[0], lin.w, lin.scale, None)
        err = (y.float() - want.float()).abs().max()
        assert err <= 2e-2 * want.float().abs().max(), float(err)
        return
    ref = xn @ lin.w.to(F64).T
    ck = Checker()
    ck._add(("gemv_rms", "fwd"), bf16_rule(f"M={M}", y, ref, _bf(ref), terms=xn.abs() @ lin.w.to(F64).abs().T))
    _report(ck)


def test_llama_decoder_generates_through_graph(C, monkeypatch):
    from alpa_b200 import ops
    from alpa_b200.model.opt_model import DecoderLM, OPTConfig
    from alpa_b200.serve import generator as gen_mod
    cfg = OPTConfig(arch="llama", vocab_size=512, hidden_size=1024, num_hidden_layers=3, num_attention_heads=8,
                    num_key_value_heads=2, ffn_dim=1536, rope_theta=500000.0)
    m = DecoderLM(cfg, device="cuda", seed=1)
    gen = gen_mod.Generator(m, 2, 96)
    seen = []
    orig = gen_mod._sample

    def record(logits, *a):
        seen.append(logits.float().clone())
        return orig(logits, *a)
    monkeypatch.setattr(gen_mod, "_sample", record)
    ids = torch.randint(4, 512, (2, 40), generator=torch.Generator().manual_seed(0))
    out = gen.generate(ids, max_new_tokens=12)
    assert gen._decode_graphs, "the decode step was not captured"
    full = gen.forward(out.sequences).float()                 # eager full forward of the generated sequence
    for t, lg in enumerate(seen):
        ref = full[:, 40 - 1 + t]
        err = (lg - ref).abs().max()
        assert err <= 0.05 * ref.abs().max() + 0.02, (t, float(err), float(ref.abs().max()))
    assert not ops.primitives.library_fallbacks()
