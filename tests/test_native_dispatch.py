"""Kernel-or-reference dispatch of every primitive on the GPU (`primitives._kernels`).

* A supported call launches an sm_90a kernel and records no library fallback.
* A call whose layout the kernel cannot take records exactly one library fallback, naming the op, and returns what the
  PyTorch reference returns with `global_config.use_native_kernels = False`.
* Without the extension every op raises, unless ALPA_B200_ALLOW_FALLBACK=1, which runs the reference.

Each case builds its inputs from a fixed seed, so two builds give the same inputs; in-place ops return the tensors they
update.
"""
import pytest
import torch

from alpa_b200 import ops
from alpa_b200.global_env import global_config
from alpa_b200.ops import primitives as P

BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn


def _rn(g, *shape, dtype=BF16):
    return torch.randn(*shape, generator=g, device="cuda").to(dtype)


def _gen():
    return torch.Generator(device="cuda").manual_seed(0)


def _ln_stats(x, eps=1e-5):
    xf = x.float()
    return xf.mean(-1), torch.rsqrt(xf.var(-1, unbiased=False) + eps)


def _ce_stats(logits, labels):
    lf = logits.float()
    mx = lf.max(1).values
    return torch.stack([mx, torch.exp(lf - mx[:, None]).sum(1), lf.gather(1, labels[:, None])[:, 0]], 1)


def _fp8_weight(g, N, K):
    w = torch.randn(N, K, generator=g, device="cuda")
    scale = w.abs().amax(1).clamp(min=1e-8) / 448.0
    return (w / scale[:, None]).to(E4M3), scale


def _route(G, S, E, C):
    """(expert, slot) of the reference top-2 routing, computed on the CPU."""
    gates = torch.softmax(torch.randn(G, S, E, generator=torch.Generator().manual_seed(1)), -1)
    return tuple(t.cuda() for t in P.moe_top2_route(gates, C))


# ---- one builder per case: () -> (() -> outputs); `M`, `H`, `D`, `V` etc. choose a supported or unsupported layout ----
def _linear(M):
    g = _gen()
    x, w, b = _rn(g, 2, M, 128), _rn(g, 96, 128), _rn(g, 96)
    return lambda: P.linear(x, w, b)


def _linear_act(M):
    g = _gen()
    x, w, b = _rn(g, 2, M, 128), _rn(g, 96, 128), _rn(g, 96)
    return lambda: P.linear_act(x, w, b, "gelu")


def _linear_dgrad(M):
    g = _gen()
    dy, w = _rn(g, 2, M, 96), _rn(g, 96, 128)
    return lambda: P.linear_dgrad(dy, w)


def _linear_dgrad_act(z_cols):
    g = _gen()
    dy, w, z = _rn(g, 128, 96), _rn(g, 96, 128), _rn(g, 128, z_cols)[:, :128]
    return lambda: P.linear_dgrad_act(dy, w, z, "gelu")


def _linear_dgrad_add(r_cols):
    g = _gen()
    dy, w, r = _rn(g, 128, 96), _rn(g, 96, 128), _rn(g, 128, r_cols)[:, :128]
    return lambda: P.linear_dgrad_add(dy, w, r)


def _linear_wgrad(M):
    g = _gen()
    dy, x = _rn(g, M, 96), _rn(g, M, 128)
    return lambda: P.linear_wgrad(dy, x)


def _linear_wgrad_out(M):
    g = _gen()
    dy, x = _rn(g, M, 96), _rn(g, M, 128)
    out = torch.zeros(96, 136, device="cuda", dtype=BF16)[:, 8:]          # a 16-byte aligned slice of a bucket
    return lambda: P._linear_wgrad_out(dy, x, out)


def _bias_grad(N):
    dy = _rn(_gen(), 128, N)
    return lambda: P.bias_grad(dy)


def _layer_norm(H):
    g = _gen()
    x, gam, bet = _rn(g, 16, H), _rn(g, H), _rn(g, H)
    return lambda: P.layer_norm(x, gam, bet, 1e-5)


def _add_layer_norm(H):
    g = _gen()
    x, r, gam, bet = _rn(g, 16, H), _rn(g, 16, H), _rn(g, H), _rn(g, H)
    return lambda: P.add_layer_norm(x, r, gam, bet, 1e-5)


def _layer_norm_bwd(H):
    g = _gen()
    dy, x, gam = _rn(g, 16, H), _rn(g, 16, H), _rn(g, H)
    mean, rstd = _ln_stats(x)
    return lambda: P.layer_norm_bwd(dy, x, gam, mean, rstd, None)


def _attention(D):
    g = _gen()
    q, k, v = (_rn(g, 2, 128, 4, D) for _ in range(3))
    return lambda: P.attention(q, k, v, D ** -0.5, True)


def _attention_bwd(D):
    g = _gen()
    q, k, v, do = (_rn(g, 2, 128, 4, D) for _ in range(4))
    o, lse = P._attn_ref(q, k, v, D ** -0.5, True)
    return lambda: P.attention_bwd(do, q, k, v, o, lse, D ** -0.5, True)


def _attention_gqa_packed(D):
    qkv = _rn(_gen(), 2, 128, 2, 4, D)
    return lambda: P.attention_gqa_packed(qkv, D ** -0.5, True)


def _attention_gqa_packed_bwd(D):
    g = _gen()
    qkv, do = _rn(g, 2, 128, 2, 4, D), _rn(g, 2, 128, 2, 2, D)
    o, lse = P._gqa_attn_ref(*P._gqa_split(qkv), D ** -0.5, True)
    return lambda: P.attention_gqa_packed_bwd(do, qkv, o, lse, D ** -0.5, True)


def _embedding(H):
    g = _gen()
    ids, wte = torch.randint(0, 1000, (4, 32), generator=g, device="cuda"), _rn(g, 1000, H)
    return lambda: P.embedding(ids, wte, 0)


def _embedding_bwd(H):
    g = _gen()
    ids = torch.randperm(1000, generator=g, device="cuda")[:128].view(4, 32)   # distinct rows: no scatter-add races
    dy = _rn(g, 4, 32, H)
    return lambda: P.embedding_bwd(ids, dy, 1000, 0)


def _decode_attention():
    g = _gen()
    q, kn, vn = _rn(g, 2, 1, 4, 3, 64).unbind(3)
    kc, vc = _rn(g, 2, 256, 4, 64), _rn(g, 2, 256, 4, 64)
    kv_len = torch.tensor([100], dtype=torch.int32, device="cuda")
    return lambda: (P.decode_attention(q, kn, vn, kc, vc, kv_len, 0.125), kc, vc)


def _attention_cached(T, D=64):
    g = _gen()
    q, kn, vn = _rn(g, 2, T, 4, 3, D).unbind(3)
    kc, vc = _rn(g, 2, 256, 4, D), _rn(g, 2, 256, 4, D)
    cache_len = torch.tensor(100, dtype=torch.int32, device="cuda")
    return lambda: (P.attention_cached_(q, kn, vn, kc, vc, cache_len, D ** -0.5), kc, vc)


def _ragged_attention():
    g = _gen()
    q, kc, vc = _rn(g, 3, 4, 64), _rn(g, 64, 4, 64), _rn(g, 64, 4, 64)
    seq_start = torch.tensor([0, 0, 20], dtype=torch.int32, device="cuda")
    ctx_len = torch.tensor([5, 6, 0], dtype=torch.int32, device="cuda")
    return lambda: P.ragged_attention(q, kc, vc, seq_start, ctx_len, 0.125, 8)


def _dropout(shape, dtype=BF16):
    x = _rn(_gen(), *shape, dtype=dtype)
    seed = torch.tensor(1234, dtype=torch.int64, device="cuda")
    return lambda: P.dropout(x, 0.3, seed, 1, list(shape), [0] * len(shape))


def _linear_decode(rows, fp8=False):
    g = _gen()
    x = _rn(g, rows, 256)
    w, scale = _fp8_weight(g, 128, 256) if fp8 else (_rn(g, 128, 256), None)
    return lambda: P.linear_decode(x, w, scale, None, "relu")


def _linear_fp8(N):
    g = _gen()
    x = _rn(g, 64, 256)
    w, scale = _fp8_weight(g, N, 256)
    return lambda: P.linear_fp8(x, w, scale, None, "gelu")


def _quantize_mxfp8():
    x = _rn(_gen(), 64, 256)
    return lambda: P.quantize_mxfp8(x)


def _linear_mxfp8(N):
    g = _gen()
    x = _rn(g, 64, 256)
    wq, wsf = (t.cuda() for t in P._quantize_mxfp8_ref(torch.randn(N, 256, generator=torch.Generator().manual_seed(2))))
    return lambda: P.linear_mxfp8(x, wq, wsf, None, "relu")


def _bmm(M):
    g = _gen()
    a, b = _rn(g, 2, M, 128), _rn(g, 2, 96, 128)
    return lambda: P.bmm(a, b, False, False)


def _moe_top2_route():
    gates = torch.softmax(torch.randn(2, 64, 8, generator=_gen(), device="cuda"), -1)
    return lambda: P.moe_top2_route(gates, 16)


def _moe_dispatch(M):
    g = _gen()
    expert, slot = _route(2, 64, 8, 16)
    x, w = _rn(g, 2, 64, M), _rn(g, 2, 64, 2)
    return lambda: P.moe_dispatch(x, expert, slot, w, 8, 16)


def _moe_combine(M):
    g = _gen()
    expert, slot = _route(2, 64, 8, 16)
    eo, w = _rn(g, 8, 32, M), _rn(g, 2, 64, 2)
    return lambda: P.moe_combine(eo, expert, slot, w)


def _moe_combine_wgrad(M):
    g = _gen()
    expert, slot = _route(2, 64, 8, 16)
    dout, eo = _rn(g, 2, 64, M), _rn(g, 8, 32, M)
    return lambda: P.moe_combine_wgrad(dout, eo, expert, slot)


def _cross_entropy(V):
    g = _gen()
    logits, labels = _rn(g, 64, V), torch.randint(0, V, (64,), generator=g, device="cuda")
    return lambda: P.cross_entropy(logits, labels, 0)


def _cross_entropy_bwd(V):
    g = _gen()
    logits, labels = _rn(g, 64, V), torch.randint(0, V, (64,), generator=g, device="cuda")
    stats, dloss = _ce_stats(logits, labels), torch.rand(64, generator=g, device="cuda")
    return lambda: P.cross_entropy_bwd(logits, labels, stats, dloss, 0)


def _fused_adamw():
    g = _gen()
    shapes = [(64, 40), (1000,)]
    masters = [_rn(g, *s, dtype=torch.float32) for s in shapes]
    ms = [_rn(g, *s, dtype=torch.float32) * 0.1 for s in shapes]
    vs = [torch.rand(s, generator=g, device="cuda") * 0.01 for s in shapes]
    params = [t.to(BF16) for t in masters]
    grads = [_rn(g, *s) for s in shapes]
    step = torch.tensor(3, device="cuda")

    def run():
        P.fused_adamw_(params, masters, ms, vs, grads, step, 1e-3, 0.9, 0.999, 1e-8, [0.01, 0.0], 1.0)
        return params + masters + ms + vs
    return run


def _tiles(x, strided):
    """Disjoint tiles of x [6, 10, 12]; strided: the last one has strided rows."""
    return [x[1:3, :, 4:8], x[0], x[3:6, :, 3] if strided else x[3:6, 2:5, :]]


def _pack_tiles(strided):
    views = _tiles(_rn(_gen(), 6, 10, 12), strided)
    return lambda: P.pack_tiles(views)


def _unpack_tiles(strided):
    flat = P.pack_tiles(_tiles(_rn(_gen(), 6, 10, 12).cpu(), strided)).cuda()
    y = torch.zeros(6, 10, 12, device="cuda", dtype=BF16)
    return lambda: (P.unpack_tiles(flat, _tiles(y, strided)), y)[1]


# name -> builder of a call the kernel takes
SUPPORTED = {
    "linear": lambda: _linear(64), "linear_act": lambda: _linear_act(64), "linear_dgrad": lambda: _linear_dgrad(64),
    "linear_dgrad_act": lambda: _linear_dgrad_act(128), "linear_dgrad_add": lambda: _linear_dgrad_add(128),
    "linear_wgrad": lambda: _linear_wgrad(128), "linear_wgrad_out": lambda: _linear_wgrad_out(128),
    "bias_grad": lambda: _bias_grad(96),
    "layer_norm": lambda: _layer_norm(256), "add_layer_norm": lambda: _add_layer_norm(256),
    "layer_norm_bwd": lambda: _layer_norm_bwd(256),
    "attention": lambda: _attention(64), "attention_bwd": lambda: _attention_bwd(64),
    "attention_gqa_packed": lambda: _attention_gqa_packed(64),
    "attention_gqa_packed_bwd": lambda: _attention_gqa_packed_bwd(64),
    "embedding": lambda: _embedding(64), "embedding_bwd": lambda: _embedding_bwd(64),
    "decode_attention": _decode_attention,
    "attention_cached_decode": lambda: _attention_cached(1), "attention_cached_prompt": lambda: _attention_cached(5),
    "ragged_attention": _ragged_attention,
    "dropout": lambda: _dropout((64, 128)), "dropout_fp32": lambda: _dropout((64, 128), torch.float32),
    "linear_decode": lambda: _linear_decode(4), "linear_decode_fp8": lambda: _linear_decode(4, fp8=True),
    "linear_fp8": lambda: _linear_fp8(128),
    "quantize_mxfp8": _quantize_mxfp8, "linear_mxfp8": lambda: _linear_mxfp8(128),
    "bmm": lambda: _bmm(64),
    "moe_top2_route": _moe_top2_route, "moe_dispatch": lambda: _moe_dispatch(128),
    "moe_combine": lambda: _moe_combine(128), "moe_combine_wgrad": lambda: _moe_combine_wgrad(128),
    "cross_entropy": lambda: _cross_entropy(1024), "cross_entropy_bwd": lambda: _cross_entropy_bwd(1024),
    "fused_adamw_": _fused_adamw,
    "pack_tiles": lambda: _pack_tiles(False), "unpack_tiles": lambda: _unpack_tiles(False),
}

# name -> (op the fallback names, builder of a call whose layout the kernel cannot take)
UNSUPPORTED = {
    "linear": ("linear", lambda: _linear(63)),
    "linear_act": ("linear_act", lambda: _linear_act(63)),
    "linear_dgrad": ("linear_dgrad", lambda: _linear_dgrad(63)),
    "linear_dgrad_act": ("linear_dgrad_act", lambda: _linear_dgrad_act(136)),
    "linear_dgrad_add": ("linear_dgrad_add", lambda: _linear_dgrad_add(136)),
    "linear_wgrad": ("linear_wgrad", lambda: _linear_wgrad(126)),
    "linear_wgrad_out": ("linear_wgrad", lambda: _linear_wgrad_out(118)),
    "bias_grad": ("bias_grad", lambda: _bias_grad(100)),
    "layer_norm": ("layer_norm", lambda: _layer_norm(8200)),
    "add_layer_norm": ("add_layer_norm", lambda: _add_layer_norm(8200)),
    "layer_norm_bwd": ("layer_norm_bwd", lambda: _layer_norm_bwd(8200)),
    "attention": ("attention", lambda: _attention(160)),
    "attention_bwd": ("attention_bwd", lambda: _attention_bwd(160)),
    "attention_gqa_packed": ("attention_gqa_packed", lambda: _attention_gqa_packed(160)),
    "attention_gqa_packed_bwd": ("attention_gqa_packed_bwd", lambda: _attention_gqa_packed_bwd(160)),
    "embedding": ("embedding", lambda: _embedding(60)),
    "embedding_bwd": ("embedding_bwd", lambda: _embedding_bwd(63)),
    "attention_cached_decode": ("attention_cached", lambda: _attention_cached(1, D=160)),
    "attention_cached_prompt": ("attention_cached", lambda: _attention_cached(5, D=160)),
    "dropout": ("dropout", lambda: _dropout((2,) * 6 + (4,))),
    "linear_decode": ("linear_decode", lambda: _linear_decode(9)),
    "linear_fp8": ("linear_fp8", lambda: _linear_fp8(100)),
    "linear_mxfp8": ("linear_mxfp8", lambda: _linear_mxfp8(100)),
    "bmm": ("bmm", lambda: _bmm(63)),
    "moe_dispatch": ("moe_dispatch", lambda: _moe_dispatch(100)),
    "moe_combine": ("moe_combine", lambda: _moe_combine(100)),
    "moe_combine_wgrad": ("moe_combine_wgrad", lambda: _moe_combine_wgrad(100)),
    "cross_entropy": ("cross_entropy", lambda: _cross_entropy(1001)),
    "cross_entropy_bwd": ("cross_entropy_bwd", lambda: _cross_entropy_bwd(1001)),
    "pack_tiles": ("pack_tiles", lambda: _pack_tiles(True)),
    "unpack_tiles": ("unpack_tiles", lambda: _unpack_tiles(True)),
}


@pytest.fixture(autouse=True)
def _own_fallback_record(monkeypatch):
    """Each test sees only the library fallbacks it records itself."""
    monkeypatch.setattr(P, "_FALLBACK_SEEN", set())


def _bits(out):
    """The outputs as a flat list of byte tensors (NaN-safe exact comparison)."""
    if isinstance(out, torch.Tensor):
        return [out.contiguous().reshape(-1).view(torch.uint8).cpu()]
    return [b for o in out for b in _bits(o)]


def _reference(build):
    global_config.use_native_kernels = False
    try:
        return _bits(build()())
    finally:
        global_config.use_native_kernels = True


def _assert_same(got, want, name):
    assert len(got) == len(want) and all(torch.equal(a, b) for a, b in zip(got, want)), \
        f"{name}: result differs from the PyTorch reference"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SUPPORTED))
def test_supported_call_launches_a_kernel(name):
    C = ops.native_module()
    run = SUPPORTED[name]()
    n0 = C.launch_count()
    run()
    torch.cuda.synchronize()
    assert C.launch_count() > n0, f"{name}: no sm_90a kernel launched"
    assert P.library_fallbacks() == [], P.library_fallbacks()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(UNSUPPORTED))
def test_unsupported_layout_records_one_fallback(name):
    op, build = UNSUPPORTED[name]
    got = _bits(build()())
    torch.cuda.synchronize()
    recorded = P.library_fallbacks()
    assert len(recorded) == 1 and recorded[0][0] == op, recorded
    _assert_same(got, _reference(build), name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SUPPORTED))
def test_missing_extension_raises_unless_fallback_allowed(name, monkeypatch):
    build = SUPPORTED[name]
    want = _reference(build)
    monkeypatch.setattr(ops, "native_available", lambda: False)
    monkeypatch.delenv("ALPA_B200_ALLOW_FALLBACK", raising=False)
    with pytest.raises(RuntimeError, match="extension is not built"):
        build()()
    monkeypatch.setenv("ALPA_B200_ALLOW_FALLBACK", "1")
    _assert_same(_bits(build()()), want, name)
