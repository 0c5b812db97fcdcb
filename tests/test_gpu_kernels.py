"""GPU checks of the kernels that tests/test_kernel_numerics.py and tests/test_gemm_numerics.py do not cover yet: the
native result against an fp32 PyTorch reference of the same op, within one `atol + rtol * |ref|` tolerance."""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"


def check(fails, name, got, ref, atol, rtol):
    """Appends a line for `name` to `fails` unless `got` is finite and |got - ref| <= atol + rtol * |ref| everywhere."""
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    bad = (err > atol + rtol * ref.abs()).sum().item()
    if bad or not torch.isfinite(got).all().item():
        fails.append(f"{name}: max_abs_err={err.max().item():.4g} ref_max={ref.abs().max().item():.4g} "
                     f"bad={bad}/{err.numel()}")


def test_native_extension_loaded():
    from alpa_b200 import ops
    assert ops.native_available(), "sm_90a extension must be built in-tree (python -m alpa_b200.ops.build)"
    assert hasattr(ops.native_module(), "gemm")


def test_embedding_fwd_numerics():
    """Token + position embedding, and a vocab shard (rows of ids outside it are zero)."""
    from alpa_b200 import ops
    C = ops.native_module()
    torch.manual_seed(0)
    fails = []
    Vv, H = 1000, 512
    wte = torch.randn(Vv, H, device=dev, dtype=torch.bfloat16)
    wpe = torch.randn(128, H, device=dev, dtype=torch.bfloat16)
    ids = torch.randint(0, Vv, (4, 128), device=dev)
    pos = torch.arange(128, device=dev).repeat(4, 1).contiguous()
    e = C.embedding_fwd(ids, pos, wte, wpe, 0)
    check(fails, "embedding fwd", e, (wte[ids].float() + wpe[pos].float()), 0.03, 1e-2)
    e2 = C.embedding_fwd(ids, None, wte[500:].contiguous(), None, 500)
    ref2 = torch.where((ids >= 500)[..., None], wte[ids].float(), torch.zeros(1, device=dev))
    check(fails, "embedding fwd vocab-parallel", e2, ref2, 1e-3, 1e-3)
    assert not fails, "\n".join(fails)


def test_adamw_numerics():
    """Three steps of the multi-tensor AdamW (fp32 and bf16 gradients, two weight decays) against torch.optim.AdamW:
    the fp32 master weights and their bf16 copies."""
    from alpa_b200 import ops
    C = ops.native_module()
    torch.manual_seed(0)
    fails = []
    ps = [torch.randn(n, device=dev) for n in (1000, 65536 * 2 + 3, 7)]
    gs = [torch.randn_like(p) for p in ps]
    gs[1] = gs[1].bfloat16()
    ms = [torch.zeros_like(p) for p in ps]
    vs = [torch.zeros_like(p) for p in ps]
    pb = [torch.empty_like(p, dtype=torch.bfloat16) for p in ps]
    ref_p = [p.clone().requires_grad_(True) for p in ps]
    opt = torch.optim.AdamW([{"params": ref_p[:2], "weight_decay": 0.01}, {"params": ref_p[2:], "weight_decay": 0.0}],
                            lr=1e-2, betas=(0.9, 0.999), eps=1e-8)
    tt, cc, *_host = C.adam_build_tables(gs, ps, ms, vs, pb, [0.01, 0.01, 0.0])
    for step in (1, 2, 3):
        for rp, g in zip(ref_p, gs):
            rp.grad = g.float().clone()
        opt.step()
        C.adamw_step(tt, cc, 1e-2, 0.9, 0.999, 1e-8, step, 1.0, None)
    for i in range(3):
        check(fails, f"adamw master[{i}]", ps[i], ref_p[i].detach(), 1e-5, 1e-4)
        check(fails, f"adamw bf16[{i}]", pb[i], ref_p[i].detach(), 1e-2, 1e-2)
    assert not fails, "\n".join(fails)


def test_moe_kernels_numerics():
    """MoE top-2 routing, dispatch, combine and combine_wgrad: native against the PyTorch path of the same op; ops.bmm
    (the expert GEMM) over the four operand majors against an fp32 matmul."""
    from alpa_b200 import ops
    from alpa_b200.global_env import global_config
    torch.manual_seed(3)
    fails = []

    def both(fn):
        out = fn()
        global_config.use_native_kernels = False
        try:
            ref = fn()
        finally:
            global_config.use_native_kernels = True
        return out, ref

    for (G, S, E, M) in [(2, 64, 4, 64), (4, 2048, 8, 1024), (3, 1000, 16, 256), (2, 4096, 128, 128)]:
        C = 2 * S // E
        gates = torch.softmax(torch.randn(G, S, E, device=dev), -1)
        (ex, sl), (ex_r, sl_r) = both(lambda: ops.moe_top2_route(gates, C))
        tag = f"G{G} S{S} E{E} M{M}"
        check(fails, f"moe route expert {tag}", ex, ex_r, 0, 0)
        check(fails, f"moe route slot {tag}", sl, sl_r, 0, 0)
        x = torch.randn(G, S, M, device=dev, dtype=torch.bfloat16)
        w = torch.rand(G, S, 2, device=dev, dtype=torch.bfloat16)
        for wt in (None, w):
            d, d_r = both(lambda: ops.moe_dispatch(x, ex_r, sl_r, wt, E, C))
            check(fails, f"moe dispatch w={wt is not None} {tag}", d, d_r, 1e-2, 1e-2)
            eo = torch.randn(E, G * C, M, device=dev, dtype=torch.bfloat16)
            o, o_r = both(lambda: ops.moe_combine(eo, ex_r, sl_r, wt))
            check(fails, f"moe combine w={wt is not None} {tag}", o, o_r, 2e-2, 2e-2)
        dw, dw_r = both(lambda: ops.moe_combine_wgrad(x, eo, ex_r, sl_r))
        check(fails, f"moe combine_wgrad {tag}", dw, dw_r, 0.5, 2e-2)
    for (B, Mm, N, K) in [(4, 256, 128, 64), (8, 1024, 2048, 1024), (3, 136, 72, 200)]:
        for ta in (False, True):
            for tb in (False, True):
                a = torch.randn((B, K, Mm) if ta else (B, Mm, K), device=dev, dtype=torch.bfloat16)
                b = torch.randn((B, K, N) if tb else (B, N, K), device=dev, dtype=torch.bfloat16)
                c = ops.bmm(a, b, ta, tb)
                ref = torch.matmul(a.float().transpose(1, 2) if ta else a.float(),
                                   b.float() if tb else b.float().transpose(1, 2))
                check(fails, f"bmm B{B} M{Mm} N{N} K{K} ta={int(ta)} tb={int(tb)}", c, ref, 0.3, 2e-2)
    assert not fails, "\n".join(fails)


def test_decode_attention_numerics():
    """decode_attention appends the new K / V row to the cache and attends over the first n rows: the output against
    the reference (append, then softmax attention in fp32), and the cache against the reference append."""
    from alpa_b200.ops import primitives as P
    torch.manual_seed(3)
    fails = []
    for (B, h, D, S_max, n) in [(1, 32, 80, 600, 513), (4, 8, 64, 256, 1), (2, 16, 128, 2100, 2048), (3, 4, 80, 128, 77)]:
        qkv = torch.randn(B, 1, h, 3, D, device=dev, dtype=torch.bfloat16)
        kc = torch.randn(B, S_max, h, D, device=dev, dtype=torch.bfloat16)
        vc = torch.randn(B, S_max, h, D, device=dev, dtype=torch.bfloat16)
        kc2, vc2 = kc.clone(), vc.clone()
        kv = torch.tensor([n], device=dev, dtype=torch.int32)
        q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
        o = P.decode_attention(q, k, v, kc, vc, kv, D ** -0.5)
        kc2[:, n - 1:n] = k
        vc2[:, n - 1:n] = v
        s_ = torch.einsum("bthd,bshd->bhts", q.float(), kc2[:, :n].float()) * D ** -0.5
        ref = torch.einsum("bhts,bshd->bthd", torch.softmax(s_, -1), vc2[:, :n].float())
        check(fails, f"decode_attention B{B} h{h} D{D} n{n}", o, ref, 0.03, 2e-2)
        check(fails, f"decode_attention cache append B{B} n{n}", torch.stack([kc, vc]), torch.stack([kc2, vc2]), 1e-6, 0)
    assert not fails, "\n".join(fails)


def test_primitives_match_reference_on_gpu():
    """The linear, LayerNorm and packed-attention primitives: native bf16 result vs the fp32 PyTorch computation."""
    from alpa_b200 import ops
    torch.manual_seed(0)
    x = torch.randn(4, 128, 256, device=dev, dtype=torch.bfloat16)
    w = torch.randn(512, 256, device=dev, dtype=torch.bfloat16) * 0.05
    b = torch.randn(512, device=dev, dtype=torch.bfloat16)
    y = ops.linear(x, w, b)
    ref = torch.nn.functional.linear(x.float(), w.float(), b.float())
    assert (y.float() - ref).abs().max() < 0.1
    dy = torch.randn_like(y)
    dx = ops.linear_dgrad(dy, w)
    assert (dx.float() - dy.float() @ w.float()).abs().max() < 0.3
    dw = ops.linear_wgrad(dy, x)
    assert (dw.float() - dy.float().reshape(-1, 512).t() @ x.float().reshape(-1, 256)).abs().max() < 1.5
    g = torch.ones(256, device=dev, dtype=torch.bfloat16)
    be = torch.zeros(256, device=dev, dtype=torch.bfloat16)
    yn, mean, rstd = ops.layer_norm(x, g, be, 1e-5)
    assert (yn.float() - torch.nn.functional.layer_norm(x.float(), (256,))).abs().max() < 0.05
    qkv = torch.randn(2, 256, 4, 3, 64, device=dev, dtype=torch.bfloat16)
    o, lse = ops.attention_qkvpacked(qkv, 0.125, False)
    q, k, v = (qkv[:, :, :, i].float().permute(0, 2, 1, 3) for i in range(3))
    ref_o = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v
    assert (o.float() - ref_o.permute(0, 2, 1, 3)).abs().max() < 0.05


def test_train_step_decreases_loss():
    import __graft_entry__ as g
    g.smoke()
